#!/usr/bin/env python
"""The reference's default decode chain for one Llama-3.1-8B GPTQ layer (+ lm_head), timed on the same H100 through
oracle/_ref (the reference's kernels recompiled for sm_90a; SURVEY.md 8d "reference side-by-side (i)", 9.8 row 2), next to
the Marlin GEMM at the layer's shapes.  TEST / MEASUREMENT INFRASTRUCTURE.  One JSON object per line."""
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_ref_golden import Ref  # noqa: E402

dev = torch.device("cuda:0")
ref = Ref(mem_bytes=6 << 30)


def layer_chain(ctx_len=128, n_rot=3, iters=96, vocab=128256):
    us, us_lm = ctypes.c_float(), ctypes.c_float()
    rc = ref.lib.zlref_time_decode_layer(4096, 32, 8, 128, 14336, ctx_len, n_rot, iters, vocab, ctypes.byref(us),
                                         ctypes.byref(us_lm))
    assert rc == 0, ref.lib.zlref_last_error()
    step_us = 32 * us.value + us_lm.value
    return dict(what="reference decode chain, Llama-3.1-8B GPTQ g128, batch 1", ctx=ctx_len, ref_gpu_layer_us=us.value,
                ref_gpu_lm_head_us=us_lm.value, ref_gpu_step_us_32_layers=step_us, ref_gpu_tokens_per_s=1e6 / step_us,
                kernels_per_layer=17)


def marlin(m, n, k):
    g = k // 128
    n_rot = max(2, int(300e6 // (n * k // 2)) + 1)
    qws = [torch.randint(-2 ** 31, 2 ** 31 - 1, (k // 8, n), dtype=torch.int32, device=dev) for _ in range(n_rot)]
    sc = (0.002 + 0.004 * torch.rand(g, n, device=dev)).half()
    x = torch.randn(m, k, device=dev).half()
    ptrs = (ctypes.c_void_p * n_rot)(*[w.data_ptr() for w in qws])
    us = ctypes.c_float()
    rc = ref.lib.zlref_time_marlin(ref.p(x), ptrs, ref.p(sc), n_rot, m, n, k, g, 40, ctypes.byref(us))
    assert rc == 0, ref.lib.zlref_last_error()
    alg = n * k / 2 + n * g * 2 + 2 * m * (n + k)
    return dict(what="reference gptq_marlin_gemm", m=m, n=n, k=k, ref_us=us.value, ref_gbs=alg / us.value / 1e3)


def main():
    if "--chain-only" in sys.argv:
        print(json.dumps(layer_chain(128)), flush=True)
        return
    for ctx in (128, 2048):
        print(json.dumps(layer_chain(ctx)), flush=True)
    for (n, k) in ((6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)):
        for m in (1, 16, 32, 128):
            print(json.dumps(marlin(m, n, k)), flush=True)


if __name__ == "__main__":
    main()
    sys.stdout.flush()
    os._exit(0)
