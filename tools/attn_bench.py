#!/usr/bin/env python
"""Decode attention timings (fp16 KV and int8 KV) at Llama-3.1-8B head shapes: CUDA events, KV buffers of all tasks
exceed L2 at the larger settings.  One JSON object per line; engineering probe."""
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
PEAKS = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
HBM = PEAKS.get("hbm_gbs", 6650.0)


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def bench(b, ctx, hq=32, hkv=8, d=128, layers_rot=4):
    """layers_rot independent KV sets are rotated so that small settings are not served from L2"""
    scale = 1.0 / np.sqrt(d)
    q = torch.randn(b, 1, hq, d, device=dev).half()
    lens = torch.full((b,), ctx, dtype=torch.int32, device=dev)
    sets16, sets8 = [], []
    for _ in range(layers_rot):
        ks = [torch.randn(ctx, hkv, d, device=dev).half() for _ in range(b)]
        vs = [torch.randn(ctx, hkv, d, device=dev).half() for _ in range(b)]
        sets16.append((ks, vs))
        kq = [torch.randint(0, 256, (ctx, hkv, d), dtype=torch.uint8, device=dev) for _ in range(b)]
        vq = [torch.randint(0, 256, (ctx, hkv, d), dtype=torch.uint8, device=dev) for _ in range(b)]
        sk = [0.01 + 0.01 * torch.rand(ctx, hkv, device=dev) for _ in range(b)]
        sv = [0.01 + 0.01 * torch.rand(ctx, hkv, device=dev) for _ in range(b)]
        sets8.append((kq, vq, sk, sv))
    from zhilight_b200 import _lib
    from zhilight_b200.ops import _p, _ptr_table, _stream, _dt
    lib = _lib.load()
    ws_bytes = lib.zl_decode_attention_workspace_bytes(b, 1, hq, d, ctx)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    o = torch.empty_like(q)
    tabs16 = [(_ptr_table(ks, dev), _ptr_table(vs, dev)) for ks, vs in sets16]
    tabs8 = [tuple(_ptr_table(x, dev) for x in st) for st in sets8]
    state = {"i": 0}

    def f16():
        ka, va = tabs16[state["i"] % layers_rot]
        state["i"] += 1
        _lib.call("zl_decode_attention", _p(q), _p(lens), _p(ka), _p(va), None, float(scale), ctx, _p(o), b, 1, hq, hkv, d, 1,
                  _p(ws), ws_bytes, _dt(q), 0, _stream())

    def i8():
        ka, va, ska, sva = tabs8[state["i"] % layers_rot]
        state["i"] += 1
        _lib.call("zl_decode_attention_kv8", _p(q), _p(lens), _p(ka), _p(va), _p(ska), _p(sva), None, float(scale), ctx, _p(o),
                  b, 1, hq, hkv, d, _p(ws), ws_bytes, _dt(o), 0, _stream())

    out = []
    for name, fn, bkv, extra in (("fp16 KV", f16, 2, 0), ("int8 KV", i8, 1, 2 * hkv * ctx * 4)):
        us = timeit(fn)
        alg = b * (2 * hkv * d * ctx * bkv + extra + hq * d * 2 * 2)
        out.append(dict(kernel="decode_attention " + name, batch=b, ctx=ctx, us=us, gbs=alg / us / 1e3, hbm_frac=alg / us / 1e3 / HBM))
    return out


if __name__ == "__main__":
    for (b, ctx) in ((1, 128), (1, 2048), (8, 2048), (32, 2048), (32, 8192)):
        for r in bench(b, ctx):
            print(json.dumps(r), flush=True)
