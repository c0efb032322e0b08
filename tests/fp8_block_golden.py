"""FP8 block-scaled activation fixture (TEST INFRASTRUCTURE): seeded inputs, the exact oracle, and the generator of
tests/golden/fp8_block_ref.npz from the reference's own nn::fp8::per_token_cast_to_fp8 (fp8_util.cu:231-322).

Cases: f16 and bf16 inputs, scales column-major (the default, DeepGEMM's layout) and row-major, M not a multiple of 4
(padded scale rows), all-zero groups (amax clamps to 1e-4), groups below the clamp, and a group whose extreme maps to
-448.  Codes and scales are exact, so the fixture is compared bit for bit.

    python -m tests.fp8_block_golden <out_dir> oracle/_ref/libzl_ref_fp8.so      (on a GPU, where build() made the library)

writes <out_dir>/fp8_block_ref.npz; with oracle/_ref/libzl_dropin_fp8.so the same calls run through the drop-in
definitions, and the drop-in's deep_gemm_fp8_block_h20_group is run on GEMM_CASES as well (keys y_*)."""
import ctypes
import os
import sys

import numpy as np

from oracle import ops as oops
from tests import fp8_block_oracle as fb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "fp8_block_ref.npz")
SHAPES = {"m5k512": (5, 512), "m1k128": (1, 128), "m36k1024": (36, 1024)}
# (M, N, K) of the drop-in GEMM check: the mma.sync route, the wgmma route, a partial last scale row
GEMM_CASES = {"m3n256k512": (3, 256, 512), "m70n320k1024": (70, 320, 1024)}


def case_input(name, tag):
    """Values of the case (already rounded to tag) as float32."""
    m, k = SHAPES[name]
    r = np.random.default_rng(k + m)
    x = r.standard_normal((m, k)) * 2.0
    x[0, :128] = 0                                          # all-zero group
    if k >= 256:
        x[-1, 128:256] *= 1e-6                              # below the clamp
        x[-1, 131] = -5.0                                   # its group's extreme: -448
    return oops._t(x, tag)


def keys():
    """(case, dtype tag, col_major, key prefix): the fixture holds <prefix>_q (codes) and <prefix>_s (scales)."""
    return [(name, tag, cm, "%s_%s_%s" % (name, tag, "col" if cm else "row"))
            for name in SHAPES for tag in ("f16", "bf16") for cm in (True, False)]


def oracle(name, tag, col_major):
    q, s = fb.quant_per_token_group(case_input(name, tag))
    return q, (s if col_major else np.ascontiguousarray(s.T))


def check(g):
    """Replay a fixture against the oracle: codes and scales bit for bit (padding scale entries are not compared)."""
    n = 0
    for name, tag, cm, key in keys():
        q, s = oracle(name, tag, cm)
        m = SHAPES[name][0]
        np.testing.assert_array_equal(g[key + "_q"], q, err_msg=key)
        gs = g[key + "_s"]
        assert gs.shape == s.shape, key
        np.testing.assert_array_equal(gs[:, :m] if cm else gs[:m], s[:, :m] if cm else s[:m], err_msg=key)
        n += 1
    return n


def gemm_operands(name):
    """Quantised activations (codes, column-major scales), e4m3 weight codes and block scales of a GEMM case."""
    m, n, k = GEMM_CASES[name]
    r = np.random.default_rng(n + k)
    xq, sx = fb.quant_per_token_group(oops._t(r.standard_normal((m, k)), "bf16"))
    wq, sw = fb.random_weight(n, k, r)
    return xq, sx, wq, sw


def main(out_dir, lib_path):
    import torch
    from oracle.gen_ref_golden import Ref
    os.makedirs(out_dir, exist_ok=True)
    ref = Ref(lib_path=lib_path)
    outs = {}
    for name, tag, cm, key in keys():
        m, k = SHAPES[name]
        ld = (m + 3) // 4 * 4
        x = ref.t(case_input(name, tag)).to(torch.float16 if tag == "f16" else torch.bfloat16)
        q = torch.empty((m, k), dtype=torch.uint8, device=ref.dev)
        s = torch.zeros((k // 128, ld) if cm else (ld, k // 128), dtype=torch.float32, device=ref.dev)
        ref._chk(ref.lib.zlfp8_per_token_cast(ref.p(x), m, k, 0 if tag == "f16" else 1, int(cm), ref.p(q), ref.p(s)))
        s = s.cpu().numpy()
        # the scale rows / columns past M are padding the reference leaves unwritten: stored as 0
        if cm:
            s[:, m:] = 0
        else:
            s[m:] = 0
        outs[key + "_q"] = q.cpu().numpy()
        outs[key + "_s"] = s
    if hasattr(ref.lib, "deep_gemm_fp8_block_h20_group"):
        dg = ref.lib.deep_gemm_fp8_block_h20_group
        for name, (m, n, k) in GEMM_CASES.items():
            xq, sx, wq, sw = (ref.t(a) for a in gemm_operands(name))
            y = torch.empty((m, n), dtype=torch.bfloat16, device=ref.dev)
            stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            rc = dg(ref.p(xq), ref.p(sx), ref.p(wq), ref.p(sw), ref.p(y), None, stream, m, n, k, 64, 1)
            assert rc == 0, (name, rc)
            # the grouped (MoE) form is not served: -1, which Fp8Block reports as an unsupported shape
            assert dg(ref.p(xq), ref.p(sx), ref.p(wq), ref.p(sw), ref.p(y), ref.p(xq), stream, m, n, k, 64, 2) == -1
            torch.cuda.synchronize()
            outs["y_" + name] = y.float().cpu().numpy()
    np.savez(os.path.join(out_dir, "fp8_block_ref.npz"), **outs)
    print("wrote", os.path.join(out_dir, "fp8_block_ref.npz"))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
    sys.stdout.flush()
    os._exit(0)      # the reference shim's statics are torn down after the CUDA driver at interpreter exit
