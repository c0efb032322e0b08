#!/usr/bin/env python
"""wgmma W4A16 kernel (k_w4a16_ts) timings at the Llama-3.1-8B projection shapes, M = 32..256, weights rotated through
> L2 worth of copies, CUDA events.  One JSON object per line; engineering probe."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zhilight_b200 import build, ops  # noqa: E402

build.build()
dev = torch.device("cuda:0")
PEAKS = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
HBM = PEAKS.get("hbm_gbs", 6650.0)
TF = PEAKS.get("bf16_tflops", 1590.0)


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


def bench(n, k, m, variant=1, graph=False):
    nbytes = (n // 32) * (k // 128) * 2128
    n_rot = max(2, int(400e6 // nbytes) + 1)
    packs = [torch.randint(0, 255, (nbytes,), dtype=torch.uint8, device=dev) for _ in range(n_rot)]
    for p in packs:                                      # sane scales: overwrite meta with small fp16 values
        v = p.view(-1, 2128)
        v[:, 2048:2112] = 0
        v[:, 2049:2112:2] = 0x1c                         # fp16 high byte 0x1c -> ~0.004
    x = torch.randn(m, k, device=dev).half()
    out = torch.empty(m, n, device=dev).half()
    if graph:
        # 20 launches (rotating weight copies) in one CUDA graph: no host launch gaps between the kernels
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            ops.w4a16_gemm_fused(x, packs[0], n, k, out=out, variant=variant)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                for i in range(20):
                    ops.w4a16_gemm_fused(x, packs[i % n_rot], n, k, out=out, variant=variant)
            us = timeit(lambda i: g.replay(), 1, iters=5, warm=2) / 20
    else:
        us = timeit(lambda i: ops.w4a16_gemm_fused(x, packs[i], n, k, out=out, variant=variant), n_rot)
    alg = nbytes + 2 * m * (k + n)
    tflops = 2.0 * m * n * k / us / 1e6
    return dict(kernel="w4a16_tc" if variant == 1 else "w4a16_v2", graph=graph, n=n, k=k, m=m, us=us, gbs=alg / us / 1e3,
                hbm_frac=alg / us / 1e3 / HBM, tflops=tflops, tensor_frac=tflops / TF)


if __name__ == "__main__":
    if len(sys.argv) >= 5 and sys.argv[1] == "--one":
        print(json.dumps(bench(int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), graph="--graph" in sys.argv)), flush=True)
        sys.exit(0)
    graph = "--graph" in sys.argv
    for (n, k) in ((6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)):
        for m in (32, 64, 128, 256):
            print(json.dumps(bench(n, k, m, graph=graph)), flush=True)
