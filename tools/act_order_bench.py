"""Act-order cost: Llama-3.1-8B GPTQ-int4 decode tok/s at batch 1 / 8 / 32 and the TTFT of a 128-token prompt, for the
synthetic sequential model against the same synthetic weights with act-order (desc_act) g_idx (alternating runs in one
process).  The act-order model stages one random g_idx per Linear input (q/k/v, o, gate/up, down) with
zl_llama_load_tensor before zl_llama_init_synthetic, which finds them as it finalises each layer.

    python tools/act_order_bench.py [--out FILE] [--reps 5] [--steps 128]
"""
import argparse
import ctypes
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.sample_bench import card  # noqa: E402

INPUTS = (("attn.project_q", "attn.project_k", "attn.project_v"), ("attn.attn_out",), ("ff.w_in", "ff.w_gated"),
          ("ff.w_out",))


def make_decoder(cfg, act_order, max_batch, max_seq, chunk, seed=0):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, max_batch=max_batch, max_seq=max_seq, prefill_chunk=chunk,
                       **cfg)
    if act_order:
        rng = np.random.default_rng(seed)
        ks = (cfg["dim_model"], cfg["num_heads"] * cfg["dim_head"], cfg["dim_model"], cfg["dim_ff"])
        for l in range(cfg["num_layers"]):
            for group, k in zip(INPUTS, ks):
                gi = np.empty(k, np.int32)
                gi[rng.permutation(k)] = np.arange(k) // 128
                for name in group:
                    _lib.check(dec.lib.zl_llama_load_tensor(dec.h, ("layers.%d.%s.g_idx" % (l, name)).encode(),
                                                            gi.ctypes.data_as(ctypes.c_void_p), 1, k, 4))
    dec.init_synthetic(seed)
    return dec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("act_order_bench needs a CUDA device")
    from zhilight_b200 import build
    from zhilight_b200.llama import MODEL_PRESETS
    build.build()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: %s" % card())
    cfg = MODEL_PRESETS["llama-3.1-8b"]
    decs = {m: make_decoder(cfg, m == "act-order", 32, 512, 128) for m in ("sequential", "act-order")}
    log("## Llama-3.1-8B GPTQ-int4 (synthetic weights, sym) decode, device-resident graph steps: %d timed steps per run, "
        "%d alternating runs per model; tok/s median (min-max)" % (args.steps, args.reps))
    rng = np.random.default_rng(0)
    for B in (1, 8, 32):
        tok = rng.integers(0, cfg["vocab_size"], size=B).astype(np.int32)
        pos = np.full(B, 128, dtype=np.int32)
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
        s, a = statistics.median(res["sequential"]), statistics.median(res["act-order"])
        log("B=%-3d sequential %.1f tok/s (%.1f-%.1f)  act-order %.1f tok/s (%.1f-%.1f)  act-order/sequential %.4f  "
            "kernels/step %d vs %d" % (B, s, min(res["sequential"]), max(res["sequential"]), a, min(res["act-order"]),
                                       max(res["act-order"]), a / s, decs["sequential"].stats(B)[1],
                                       decs["act-order"].stats(B)[1]))
    log("## TTFT of a 128-token prompt (one chunked-prefill pass of 128 tokens, host clock to the returned token), "
        "ms median (min-max) of %d alternating runs" % (2 * args.reps))
    prompt = rng.integers(0, cfg["vocab_size"], size=128).astype(np.int32)
    res = {m: [] for m in decs}
    for r in range(2 * args.reps + 1):
        for mode, dec in decs.items():
            dec.sync()
            t0 = time.perf_counter()
            dec.prefill(0, prompt)
            ms = (time.perf_counter() - t0) * 1000.0
            if r:   # the first pass warms up
                res[mode].append(ms)
    s, a = statistics.median(res["sequential"]), statistics.median(res["act-order"])
    log("sequential %.2f ms (%.2f-%.2f)  act-order %.2f ms (%.2f-%.2f)  act-order/sequential %.4f"
        % (s, min(res["sequential"]), max(res["sequential"]), a, min(res["act-order"]), max(res["act-order"]), a / s))
    for dec in decs.values():
        dec.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
