"""int8 KV cache cost and gain: Llama-3.1-8B GPTQ-int4 (synthetic weights) decode tok/s with the fp16 cache against the int8
cache (LlamaDecoder(kv_cache_dtype="int8")), batch 1 / 8 / 32 at contexts 256 / 2048 filled with zl_llama_prefill,
alternating runs of the two models in one process; then tools/attn_bench.py's fp16-vs-int8 attention kernels at the same
shapes.  KV bytes per step are algorithmic (from the shapes), not measured.

    python tools/kv8_bench.py [--out FILE] [--reps 5] [--steps 64]
"""
import argparse
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.sample_bench import card  # noqa: E402

BATCHES = (1, 8, 32)
CTXS = (256, 2048)


def kv_bytes_per_step(cfg, B, ctx, kv8):
    """bytes of K and V one decode step reads: every layer, every task, ctx cached rows (+ one fp32 scale per row and kv
    head of K and of V for the int8 cache)."""
    per_row = cfg["num_kv_heads"] * (cfg["dim_head"] + 4 if kv8 else 2 * cfg["dim_head"])
    return 2.0 * cfg["num_layers"] * B * ctx * per_row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("kv8_bench needs a CUDA device")
    from zhilight_b200 import build
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    build.build()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: %s" % card())
    cfg = MODEL_PRESETS["llama-3.1-8b"]
    max_b, max_ctx = max(BATCHES), max(CTXS)
    max_seq = max_ctx + args.warmup + args.steps + 64
    decs = {}
    for mode in ("fp16 KV", "int8 KV"):
        dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, max_batch=max_b, max_seq=max_seq, prefill_chunk=512,
                           kv_cache_dtype="int8" if mode == "int8 KV" else None, **cfg)
        dec.init_synthetic(0)
        decs[mode] = dec
    rng = np.random.default_rng(0)
    prompts = rng.integers(0, cfg["vocab_size"], size=(max_b, max_ctx)).astype(np.int32)
    for dec in decs.values():     # every task's rows 0 .. 2047; a run at context c decodes at positions c, c + 1, ...
        for t in range(max_b):
            dec.prefill(t, prompts[t])
    wbytes = decs["fp16 KV"].stats(1)[0]
    log("## Llama-3.1-8B GPTQ-int4 (synthetic weights, sym) decode, device-resident graph steps: %d timed steps per run after "
        "%d warm-up steps, %d alternating runs per model; tok/s median (min-max).  Weights + lm_head %.2f GB per step; KV "
        "GB per step algorithmic at the run's starting context" % (args.steps, args.warmup, args.reps, wbytes / 1e9))
    for ctx in CTXS:
        for B in BATCHES:
            tok = rng.integers(0, cfg["vocab_size"], size=B).astype(np.int32)
            pos = np.full(B, ctx, dtype=np.int32)
            res = {m: [] for m in decs}
            for _ in range(args.reps):
                for mode, dec in decs.items():
                    st = torch.cuda.ExternalStream(dec.stream())
                    dec.set_state(tok, pos)
                    for _ in range(args.warmup):
                        dec.step_device(B)
                    dec.sync()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    for _ in range(args.steps):
                        dec.step_device(B)
                    e1.record(st)
                    e1.synchronize()
                    res[mode].append(B * args.steps * 1000.0 / e0.elapsed_time(e1))
            f, i = statistics.median(res["fp16 KV"]), statistics.median(res["int8 KV"])
            log("B=%-3d ctx=%-5d fp16 KV %.1f tok/s (%.1f-%.1f)  int8 KV %.1f tok/s (%.1f-%.1f)  int8/fp16 %.4f  "
                "KV GB/step %.3f vs %.3f  kernels/step %d vs %d"
                % (B, ctx, f, min(res["fp16 KV"]), max(res["fp16 KV"]), i, min(res["int8 KV"]), max(res["int8 KV"]), i / f,
                   kv_bytes_per_step(cfg, B, ctx, False) / 1e9, kv_bytes_per_step(cfg, B, ctx, True) / 1e9,
                   decs["fp16 KV"].stats(B)[1], decs["int8 KV"].stats(B)[1]))
    for dec in decs.values():
        dec.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    from tools import attn_bench
    log("## one attention launch (tools/attn_bench.py: 32 q heads, 8 kv heads, d = 128, 4 rotating KV sets), us per call; "
        "algorithmic GB/s")
    for ctx in CTXS:
        for B in BATCHES:
            r16, r8 = attn_bench.bench(B, ctx)
            log("B=%-3d ctx=%-5d fp16 KV %.2f us (%.0f GB/s)  int8 KV %.2f us (%.0f GB/s)  int8/fp16 time %.3f"
                % (B, ctx, r16["us"], r16["gbs"], r8["us"], r8["gbs"], r8["us"] / r16["us"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
