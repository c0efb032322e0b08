"""MLA decode attention fixture (TEST INFRASTRUCTURE): seeded inputs, the fp32 oracle, and the generator of
tests/golden/mla_ref.npz from the reference's own kernels.

The reference's MLA search path calls multi_query_attention_rag_buffer with dim_head 576, one latent head and a 512-wide
output (src/nn/attention/multi_head_latent_attention.cpp:1053-1068).  oracle.ops.decode_attention writes an output as wide
as q, so the oracle here passes V zero-padded from 512 to 576 columns and keeps the first 512 output columns: the padding
adds exact zeros and leaves the softmax untouched.

    python -m tests.mla_golden <out_dir> oracle/_ref/libzl_ref_mla.so      (on a GPU, where build() made the library)

writes <out_dir>/mla_ref.npz; with oracle/_ref/libzl_dropin_mla.so the same calls run through the drop-in definitions."""
import ctypes
import os
import sys

import numpy as np

from oracle import ops as oops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "mla_ref.npz")
TOL = {"f16": 1e-3, "bf16": 4e-3}


def mla_oracle(q, kvs, lens, masks, scale, tag):
    """q (B, len_q, H, 576); kvs list of (len_b, 1, 576) latent caches (already rounded to tag); -> (B, len_q, H, 512)."""
    vs = [np.concatenate([kv[..., :512], np.zeros(kv.shape[:-1] + (64,), np.float32)], -1) for kv in kvs]
    return oops.decode_attention(q, kvs, vs, lens, masks, scale, q.shape[2], tag)[..., :512]


def case_mla():
    """Sub-cases {name: (H, len_q, lens, mask kind)}: H 16 and 128, len_q 1 and 2 (causal), max_len_buf at most 1024 and
    above it with a short task beside a long one.  Values are float32, rounded to fp16 / bf16 where they are used."""
    r = np.random.default_rng(151)
    subs = {"h16": (16, 1, [300, 77, 1024], "random"), "h16_causal": (16, 2, [2500, 400], "causal"),
            "h128": (128, 1, [1100], "random")}
    cases = {}
    for name, (h, len_q, lens, kind) in subs.items():
        q = r.standard_normal((len(lens), len_q, h, 576)).astype(np.float32)
        kvs = [r.standard_normal((lb, 1, 576)).astype(np.float32) for lb in lens]
        masks = []
        for lb in lens:
            m = np.ones((len_q, lb), np.int8)
            if kind == "causal":
                for i in range(len_q):
                    m[i, lb - len_q + i + 1:] = 0
            else:
                m[:, r.permutation(lb)[: lb // 7]] = 0
            masks.append(m)
        cases[name] = dict(q=q, kvs=kvs, masks=masks, lens=np.array(lens, np.int32), h=h, len_q=len_q)
    return dict(cases=cases, scale=float(1.0 / np.sqrt(192.0)))


def keys():
    """(sub-case name, dtype tag, fixture key): bf16 keys end in _bf16."""
    return [(name, tag, "out_%s" % name + ("_bf16" if tag == "bf16" else ""))
            for name in case_mla()["cases"] for tag in ("f16", "bf16")]


def check(g):
    """Replay a fixture against the oracle; returns {key: rel L2}."""
    c = case_mla()
    errs = {}
    for name, tag, key in keys():
        sc = c["cases"][name]
        kvs = [oops._t(kv, tag) for kv in sc["kvs"]]
        ref = mla_oracle(oops._t(sc["q"], tag), kvs, sc["lens"], sc["masks"], c["scale"], tag)
        a, b = np.asarray(g[key], np.float64), np.asarray(ref, np.float64)
        errs[key] = float(np.linalg.norm(a - b) / np.linalg.norm(b))
        assert errs[key] < TOL[tag], (key, errs[key])
    return errs


def mla_call(ref, q, lens, kvs, mask_flat, scale):
    """One zlref_mqa_rag_buffer_mla call through `ref` (an oracle.gen_ref_golden.Ref over libzl_ref_mla.so or
    libzl_dropin_mla.so); q (B, len_q, H, 576), kvs per-task (len, 576) device tensors."""
    import torch
    b, len_q, hq, _ = q.shape
    table = torch.tensor([t.data_ptr() for t in kvs], dtype=torch.int64, device=ref.dev)
    out = torch.empty((b, len_q, hq, 512), dtype=q.dtype, device=ref.dev)
    ref._chk(ref.lib.zlref_mqa_rag_buffer_mla(ref.p(q), ref.p(lens), ref.p(table), ref.p(mask_flat),
                                              ctypes.c_size_t(mask_flat.numel()), ctypes.c_float(scale),
                                              int(lens.max().item()), b, len_q, hq, 0 if q.dtype == torch.float16 else 1,
                                              ref.p(out)))
    return out


def main(out_dir, lib_path):
    import torch
    from oracle.gen_ref_golden import Ref
    os.makedirs(out_dir, exist_ok=True)
    ref = Ref(lib_path=lib_path)
    c = case_mla()
    outs = {}
    for name, tag, key in keys():
        sc = c["cases"][name]
        dt = torch.float16 if tag == "f16" else torch.bfloat16
        mask = ref.t(np.concatenate([m.reshape(-1) for m in sc["masks"]]))
        kvs = [ref.t(kv.reshape(-1, 576)).to(dt) for kv in sc["kvs"]]
        out = mla_call(ref, ref.t(sc["q"]).to(dt), ref.t(sc["lens"]), kvs, mask, c["scale"])
        # bf16 outputs are kept as fp16: exact for these magnitudes, and half the bytes of fp32
        outs[key] = out.half().cpu().numpy()
    np.savez(os.path.join(out_dir, "mla_ref.npz"), **outs)
    print("wrote", os.path.join(out_dir, "mla_ref.npz"))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
    sys.stdout.flush()
    os._exit(0)      # the reference shim's statics are torn down after the CUDA driver at interpreter exit
