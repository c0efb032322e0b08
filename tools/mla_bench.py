#!/usr/bin/env python
"""MLA decode attention (zl_mla_decode_attention) kernel time at H 16 / 128, len_q 1 / 2, B 1 / 8 / 32 / 64 and contexts
1024 / 4096 / 16384, against both rooflines of an H100 SXM (3.35 TB/s HBM3, 989 TFLOP/s dense fp16), and beside the
reference's multi_query_attention_rag_buffer(576) (oracle/_ref/libzl_ref_mla.so over the reference's kernels) when
that library is built.

CUDA events over 50 launches after warm-up; the two implementations alternate, three rounds each, and the median is
reported.  Several latent-cache sets are rotated so that a shape's caches are not served from the 50 MB L2.  Algorithmic
bytes = B ctx 1152 + q + out + mask; FLOPs = 2 B len_q H ctx 1088.  Writes profiles/mla_bench.txt (or the path given)."""
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zhilight_b200 import _lib, build, ops  # noqa: E402
from zhilight_b200.ops import _dt, _p, _ptr_table, _stream  # noqa: E402

HBM_BPS, FLOPS = 3.35e12, 989e12
REF = os.path.join(ROOT, "oracle", "_ref", "libzl_ref_mla.so")
ITERS, ROUNDS = 50, 3


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def main(out_path):
    build.build()
    dev = torch.device("cuda:0")
    ref = None
    if os.path.exists(REF):
        from oracle.gen_ref_golden import Ref
        ref = Ref(mem_bytes=4 << 30, lib_path=REF)
    lib = _lib.load()
    lines = ["# MLA decode attention: card %s" % card(),
             "# kernel us = CUDA events, median of %d alternating rounds x %d launches; ref = reference "
             "multi_query_attention_rag_buffer(576)%s" % (ROUNDS, ITERS, "" if ref else " (not built: not measured)")]
    print("\n".join(lines), flush=True)
    scale = 1.0 / 192 ** 0.5
    for h in (16, 128):
        for len_q in (1, 2):
            for b in (1, 8, 32, 64):
                for ctx in (1024, 4096, 16384):
                    kv_bytes = b * ctx * 1152
                    n_rot = max(1, min(8, int(200e6 // kv_bytes) + 1))
                    sets = [[torch.randn(ctx, 576, device=dev).half() for _ in range(b)] for _ in range(n_rot)]
                    tabs = [_ptr_table(s, dev) for s in sets]
                    q = torch.randn(b, len_q, h, 576, device=dev).half()
                    lens = torch.full((b,), ctx, dtype=torch.int32, device=dev)
                    mask = torch.ones(b * len_q * ctx, dtype=torch.int8, device=dev) if len_q > 1 else None
                    if mask is not None:   # causal over the len_q new rows
                        m = mask.view(b, len_q, ctx)
                        for i in range(len_q):
                            m[:, i, ctx - len_q + i + 1:] = 0
                    out = torch.empty(b, len_q, h, 512, device=dev).half()
                    wsb = lib.zl_mla_decode_attention_workspace_bytes(b, len_q, h, ctx)
                    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev)
                    state = {"i": 0}

                    def ours():
                        ka = tabs[state["i"] % n_rot]
                        state["i"] += 1
                        _lib.call("zl_mla_decode_attention", _p(q), _p(lens), _p(ka), _p(mask), float(scale), ctx, _p(out),
                                  b, len_q, h, _p(ws), wsb, _dt(q), 0, _stream())

                    def time_ours():
                        for _ in range(3):
                            ours()
                        torch.cuda.synchronize()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(ITERS):
                            ours()
                        e1.record()
                        e1.synchronize()
                        return e0.elapsed_time(e1) * 1e3 / ITERS

                    def time_ref():
                        rmask = mask if mask is not None else torch.ones(b * len_q * ctx, dtype=torch.int8, device=dev)
                        tab_ptrs = (ctypes.c_void_p * n_rot)(*[t.data_ptr() for t in tabs])
                        us = ctypes.c_float()
                        rc = ref.lib.zlref_time_mqa_rag_buffer_mla(ref.p(q), ref.p(lens), tab_ptrs, n_rot, ref.p(rmask),
                                                                    ctypes.c_size_t(rmask.numel()), ctypes.c_float(scale),
                                                                    ctx, b, len_q, h, 0, ref.p(out), ITERS, ctypes.byref(us))
                        torch.cuda.synchronize()
                        return us.value if rc == 0 else float("nan")

                    t_ours, t_ref = [], []
                    for _ in range(ROUNDS):
                        t_ours.append(time_ours())
                        if ref is not None:
                            t_ref.append(time_ref())
                    us = sorted(t_ours)[ROUNDS // 2]
                    ref_us = sorted(t_ref)[ROUNDS // 2] if t_ref else None
                    alg_bytes = kv_bytes + b * len_q * h * (576 + 512) * 2 + (b * len_q * ctx if mask is not None else 0)
                    flops = 2.0 * b * len_q * h * ctx * 1088
                    t_mem, t_mma = alg_bytes / HBM_BPS * 1e6, flops / FLOPS * 1e6
                    row = dict(H=h, len_q=len_q, B=b, ctx=ctx, us=round(us, 2), tb_s=round(alg_bytes / us / 1e6, 3),
                               hbm_frac=round(t_mem / us, 3), tflops=round(flops / us / 1e6, 1),
                               mma_frac=round(t_mma / us, 3), bound="hbm" if t_mem >= t_mma else "mma",
                               roofline_frac=round(max(t_mem, t_mma) / us, 3),
                               ref_us=round(ref_us, 2) if ref_us else None,
                               speedup=round(ref_us / us, 2) if ref_us else None)
                    print(json.dumps(row), flush=True)
                    lines.append(json.dumps(row))
                    del sets, tabs
                    torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "mla_bench.txt"))
    sys.stdout.flush()
    os._exit(0)      # the reference shim's statics are torn down after the CUDA driver at interpreter exit
