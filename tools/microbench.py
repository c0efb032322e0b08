#!/usr/bin/env python
"""Kernel-level timings on one H100 (CUDA events, L2-cold by rotating through weight copies > L2).
Writes one JSON object per line.  Not the bench contract -- an engineering probe."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zhilight_b200 import build, ops  # noqa: E402

build.build()
dev = torch.device("cuda:0")
PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
    os.path.join(ROOT, "MEASURED_PEAKS.json")) else 6650.0


def timeit(fn, n_rot, iters=20, warm=3):
    for i in range(warm):
        fn(i % n_rot)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i % n_rot)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3          # us


def bench_w4(n, k, m, epi=0, pdl=False):
    nbytes = (n // 32) * (k // 128) * 2128
    n_rot = max(2, int(400e6 // nbytes) + 1)
    packs = [torch.randint(0, 255, (nbytes,), dtype=torch.uint8, device=dev) for _ in range(n_rot)]
    for p in packs:                                      # sane scales: overwrite meta with small fp16 values
        v = p.view(-1, 2128)
        v[:, 2048:2112] = torch.full((64,), 0, dtype=torch.uint8, device=dev)
        v[:, 2049:2112:2] = 0x1c                         # fp16 high byte 0x1c -> ~0.004
    x = torch.randn(m, k, device=dev).half()
    res = torch.zeros(m, n, device=dev).half()
    out = torch.empty(m, n // 2 if epi == 1 else n, device=dev).half()
    us = timeit(lambda i: ops.w4a16_gemm(x, packs[i], n, k, residual=res if epi == 2 else None, epilogue=epi, pdl=pdl,
                                         out=out), n_rot)
    alg = nbytes + 2 * m * (k + n)
    return dict(kernel="w4a16", n=n, k=k, m=m, epi=epi, pdl=pdl, us=us, gbs=alg / us / 1e3, frac=alg / us / 1e3 / PEAK)


def bench_dense(n, k, m, dtype=torch.float16):
    nbytes = n * k * 2
    n_rot = max(2, int(400e6 // nbytes) + 1)
    ws = [torch.randn(n, k, device=dev).to(dtype) for _ in range(n_rot)]
    x = torch.randn(m, k, device=dev).to(dtype)
    us = timeit(lambda i: ops.dense_gemm_skinny(x, ws[i], out_dtype=torch.float32), n_rot)
    alg = nbytes + 2 * m * k + 4 * m * n
    return dict(kernel="dense", n=n, k=k, m=m, us=us, gbs=alg / us / 1e3, frac=alg / us / 1e3 / PEAK)


def bench_attn(b, ctx, hq=32, hkv=8, d=128):
    ks = [torch.randn(ctx, hkv, d, device=dev).half() for _ in range(b)]
    vs = [torch.randn(ctx, hkv, d, device=dev).half() for _ in range(b)]
    q = torch.randn(b, 1, hq, d, device=dev).half()
    lens = torch.full((b,), ctx, dtype=torch.int32, device=dev)
    ka = torch.tensor([t.data_ptr() for t in ks], dtype=torch.int64, device=dev)
    va = torch.tensor([t.data_ptr() for t in vs], dtype=torch.int64, device=dev)
    import ctypes
    from zhilight_b200 import _lib
    out = torch.empty_like(q)
    wsb = _lib.load().zl_decode_attention_workspace_bytes(b, 1, hq, d, ctx)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())

    def run(_):
        _lib.call("zl_decode_attention", P(q), P(lens), P(ka), P(va), None, float(d ** -0.5), ctx, P(out), b, 1, hq, hkv,
                  d, 1, P(ws), wsb, 0, 0, st)
    us = timeit(run, 1)
    alg = 2 * b * ctx * hkv * d * 2
    return dict(kernel="decode_attn", b=b, ctx=ctx, us=us, gbs=alg / us / 1e3, frac=alg / us / 1e3 / PEAK)


def bench_norm(t, d):
    x = torch.randn(t, d, device=dev).half()
    w = torch.ones(d, device=dev).half()
    us = timeit(lambda i: ops.rmsnorm(x, w, 1e-5), 1)
    return dict(kernel="rmsnorm", t=t, d=d, us=us)


if __name__ == "__main__":
    rows = []
    for m in (1, 4, 8, 16, 32):
        for (n, k, epi) in ((6144, 4096, 0), (4096, 4096, 2), (28672, 4096, 1), (4096, 14336, 2)):
            rows.append(bench_w4(n, k, m, epi))
            print(json.dumps(rows[-1]), flush=True)
    rows.append(bench_w4(28672, 4096, 1, 1, pdl=True))
    print(json.dumps(rows[-1]), flush=True)
    for m in (1, 8, 32):
        rows.append(bench_dense(128256, 4096, m))
        print(json.dumps(rows[-1]), flush=True)
    for (b, ctx) in ((1, 128), (1, 2048), (8, 2048), (32, 2048), (32, 128)):
        rows.append(bench_attn(b, ctx))
        print(json.dumps(rows[-1]), flush=True)
    for t in (1, 32):
        rows.append(bench_norm(t, 4096))
        print(json.dumps(rows[-1]), flush=True)
