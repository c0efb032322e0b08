#!/usr/bin/env python
"""wgmma W4A16 kernel with its fused epilogues (none / residual / SwiGLU) and with / without programmatic dependent launch,
CUDA-graph timing of 20 back-to-back launches on rotating weights.  Engineering probe: explains the gap between the plain
GEMM microbench and the in-chain prefill GEMMs."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zhilight_b200 import build, ops  # noqa: E402

build.build()
dev = torch.device("cuda:0")


def run(n, k, m, epi, pdl):
    nbytes = (n // 32) * (k // 128) * 2128
    n_rot = max(2, int(400e6 // nbytes) + 1)
    packs = [torch.randint(0, 255, (nbytes,), dtype=torch.uint8, device=dev) for _ in range(n_rot)]
    for p in packs:
        v = p.view(-1, 2128)
        v[:, 2048:2112] = 0
        v[:, 2049:2112:2] = 0x1c
    x = torch.randn(m, k, device=dev).half()
    n_out = n // 2 if epi == ops.EPI_SWIGLU else n
    out = torch.empty(m, n_out, device=dev).half()
    res = torch.randn(m, n, device=dev).half() if epi == ops.EPI_RESIDUAL else None
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ops.w4a16_gemm_fused(x, packs[0], n, k, out=out, variant=1, residual=res, epilogue=epi, pdl=pdl)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for i in range(20):
                ops.w4a16_gemm_fused(x, packs[i % n_rot], n, k, out=out, variant=1, residual=res, epilogue=epi, pdl=pdl)
        for _ in range(2):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            g.replay()
        e1.record()
        e1.synchronize()
    return e0.elapsed_time(e1) / 100 * 1e3


if __name__ == "__main__":
    names = {ops.EPI_NONE: "none", ops.EPI_RESIDUAL: "residual", ops.EPI_SWIGLU: "swiglu"}
    for m in (128, 32):
        for (n, k, epis) in ((4096, 4096, (ops.EPI_NONE, ops.EPI_RESIDUAL)), (28672, 4096, (ops.EPI_NONE, ops.EPI_SWIGLU)),
                             (4096, 14336, (ops.EPI_NONE, ops.EPI_RESIDUAL))):
            for epi in epis:
                for pdl in (False, True):
                    us = run(n, k, m, epi, pdl)
                    print(json.dumps(dict(n=n, k=k, m=m, epilogue=names[epi], pdl=pdl, us=round(us, 1))), flush=True)
