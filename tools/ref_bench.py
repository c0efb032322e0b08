#!/usr/bin/env python
"""Reference kernels (recompiled for sm_90a, oracle/_ref) vs ours on the same H100: W4A16 GEMV at the
Llama-3.1-8B shapes.  CUDA events, weights rotated through > L2 worth of copies.  One JSON object per line."""
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_ref_golden import Ref  # noqa: E402
from zhilight_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
ref = Ref(mem_bytes=1 << 30)


def main():
    for (n, k) in ((6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)):
        g = k // 128
        nbytes = n * k // 2
        n_rot = max(2, int(300e6 // nbytes) + 1)
        qws = [torch.randint(-2 ** 31, 2 ** 31 - 1, (n, k // 8), dtype=torch.int32, device=dev) for _ in range(n_rot)]
        qz = torch.randint(0, 16, (n, g), dtype=torch.uint8, device=dev)
        sc = (0.002 + 0.004 * torch.rand(n, g, device=dev)).half()
        packs = [ops.w4_pack(w, qz, sc) for w in qws]
        ptrs = (ctypes.c_void_p * n_rot)(*[w.data_ptr() for w in qws])
        for m in (1, 8, 32):
            x = torch.randn(m, k, device=dev).half()
            out = torch.empty(m, n, device=dev).half()
            us = ctypes.c_float()
            rc = ref.lib.zlref_time_gptq_gemv(ref.p(x), ptrs, ref.p(qz), ref.p(sc), n_rot, 0, m, n, k, g, ref.p(out), 50,
                                              ctypes.byref(us))
            assert rc == 0, ref.lib.zlref_last_error()
            for i in range(3):
                ops.w4a16_gemm(x, packs[i % n_rot], n, k, out=out)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(50):
                ops.w4a16_gemm(x, packs[i % n_rot], n, k, out=out)
            e1.record()
            e1.synchronize()
            ours = e0.elapsed_time(e1) * 1e3 / 50
            alg = nbytes + n * g * 2.5 + 2 * m * (n + k)
            print(json.dumps(dict(n=n, k=k, m=m, ref_us=us.value, ours_us=ours, ref_gbs=alg / us.value / 1e3,
                                  ours_gbs=alg / ours / 1e3, speedup=us.value / ours)), flush=True)


if __name__ == "__main__":
    main()
    sys.stdout.flush()
    os._exit(0)
