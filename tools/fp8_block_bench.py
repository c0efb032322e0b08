"""FP8 block-scaled Linear (QuantType 10) against per-tensor FP8 (QuantType 7) on the same weight bytes.

1. One Linear (activation quant launch + GEMM) at the Llama-3.1-8B shapes and M = 1 / 8 / 32 / 33 / 256 / 2048:
   ops.fp8_block_linear against ops.fp8_linear, CUDA events over many calls; for M <= 32 the weight bytes over time as a
   share of 3.35 TB/s, for M = 2048 the FLOPs over time as a share of 1979 TFLOP/s (H100 SXM data sheet, dense FP8).
2. Llama-3.1-8B decode tok/s at batch 1 / 8 / 32 (synthetic weights, device-resident graph steps) and TTFT of a 128-token
   prompt, type 10 against type 7 in alternating runs in one process.

    python tools/fp8_block_bench.py [--out FILE] [--reps 5] [--steps 64]
"""
import argparse
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.sample_bench import card  # noqa: E402

SHAPES = (("qkv", 6144, 4096), ("o", 4096, 4096), ("gate_up", 28672, 4096), ("down", 4096, 14336))
MS = (1, 8, 32, 33, 256, 2048)
BATCHES = (1, 8, 32)
HBM_BPS, FP8_FLOPS = 3.35e12, 1979e12


def time_calls(fn, iters):
    import torch
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters   # us per call


def linear_bench(log, reps):
    import torch
    from zhilight_b200 import ops
    log("## one Linear incl. its activation quant launch, us per call (median of %d runs of 50-200 calls); weights "
        "rotate over 4 copies so that the weight stream comes from HBM" % reps)
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, n, k in SHAPES:
        ws = [torch.randint(0, 256, (n, k), dtype=torch.uint8, device="cuda", generator=g) & 0xBF for _ in range(4)]
        sblk = [torch.rand(((n + 127) // 128, k // 128), device="cuda", generator=g) * 0.05 + 0.01 for _ in range(4)]
        sten = torch.tensor([0.03], device="cuda")
        for m in MS:
            x = torch.randn((m, k), device="cuda", generator=g).half()
            state = {"i": 0}

            def blk():
                i = state["i"] = (state["i"] + 1) & 3
                ops.fp8_block_linear(x, ws[i], sblk[i])

            def ten():
                i = state["i"] = (state["i"] + 1) & 3
                ops.fp8_linear(x, ws[i], sten)

            iters = 200 if m <= 33 else 50
            # the per-tensor activation quant of type 7 is one CTA-cooperative launch for at most 4 Mi elements
            has7 = m * k <= (1 << 22)
            tb, tt = [], []
            for _ in range(reps):
                tb.append(time_calls(blk, iters))
                if has7:
                    tt.append(time_calls(ten, iters))
            b = statistics.median(tb)
            t = statistics.median(tt) if has7 else float("nan")
            t7 = ("type7 %8.2f us  10/7 time %.3f" % (t, b / t)) if has7 else "type7 n/a (M*K > 4 Mi)"
            if m <= 32:
                share = "weights %.1f%% of 3.35 TB/s (type 7: %.1f%%)" % (100 * n * k / (b * 1e-6) / HBM_BPS,
                                                                          100 * n * k / (t * 1e-6) / HBM_BPS)
            elif m == 2048:
                share = "%.1f%% of 1979 TFLOP/s" % (100 * 2.0 * m * n * k / (b * 1e-6) / FP8_FLOPS)
            else:
                share = ""
            log("%-7s N=%-5d K=%-5d M=%-4d type10 %8.2f us  %s  %s" % (name, n, k, m, b, t7, share))
        del ws, sblk
        torch.cuda.empty_cache()


def decode_bench(log, reps, steps, warmup):
    import torch
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    cfg = MODEL_PRESETS["llama-3.1-8b"]
    max_b = max(BATCHES)
    decs = {}
    for q in (7, 10):
        dec = LlamaDecoder(quant_type=q, max_batch=max_b, max_seq=512, prefill_chunk=128, **cfg)
        dec.init_synthetic(0)
        decs[q] = dec
    log("## Llama-3.1-8B decode (synthetic weights, f16), device-resident graph steps at context 128: %d timed steps per "
        "run after %d warm-up steps, %d alternating runs per model; tok/s median (min-max)" % (steps, warmup, reps))
    rng = np.random.default_rng(0)
    prompt = rng.integers(0, cfg["vocab_size"], size=128).astype(np.int32)
    ttft = {q: [] for q in decs}
    for _ in range(reps):
        for q, dec in decs.items():
            for t in range(max_b):
                dec.sync()
                t0 = time.perf_counter()
                dec.prefill(t, prompt)      # returns the next token: ends in a device synchronise
                if t < 4:
                    ttft[q].append((time.perf_counter() - t0) * 1e3)
    goal = True
    for B in BATCHES:
        tok = rng.integers(0, cfg["vocab_size"], size=B).astype(np.int32)
        pos = np.full(B, 128, dtype=np.int32)
        res = {q: [] for q in decs}
        for _ in range(reps):
            for q, dec in decs.items():
                st = torch.cuda.ExternalStream(dec.stream())
                dec.set_state(tok, pos)
                for _ in range(warmup):
                    dec.step_device(B)
                dec.sync()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                for _ in range(steps):
                    dec.step_device(B)
                e1.record(st)
                e1.synchronize()
                res[q].append(B * steps * 1000.0 / e0.elapsed_time(e1))
        a, b = statistics.median(res[7]), statistics.median(res[10])
        goal &= b >= 0.95 * a
        log("B=%-3d type7 %.1f tok/s (%.1f-%.1f)  type10 %.1f tok/s (%.1f-%.1f)  10/7 %.4f  goal >= 0.95: %s"
            % (B, a, min(res[7]), max(res[7]), b, min(res[10]), max(res[10]), b / a, "met" if b >= 0.95 * a else "MISSED"))
    a, b = statistics.median(ttft[7]), statistics.median(ttft[10])
    log("TTFT(128) prefill of one 128-token prompt (host clock, ends in a synchronise): type7 %.2f ms  type10 %.2f ms  "
        "10/7 %.3f" % (a, b, b / a))
    log("decode goal (type 10 >= 0.95x type 7 tok/s at every batch): %s" % ("met" if goal else "MISSED"))
    for dec in decs.values():
        dec.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fp8_block_bench needs a CUDA device")
    from zhilight_b200 import build
    build.build()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: %s" % card())
    linear_bench(log, args.reps)
    decode_bench(log, args.reps, args.steps, args.warmup)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
