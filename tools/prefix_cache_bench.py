"""Prompt prefix cache: time to first token with and without the cache, and the block copy that serves it.

Llama-3.1-8B GPTQ-int4 (synthetic weights, sym), prefill_chunk 512, 128-token blocks, fp16 and int8 KV caches.  For a
shared prefix of 512 / 2048 / 4096 tokens followed by 64 new tokens:
  - TTFT cold: zl_llama_prefill of the whole prompt (task 0); cached: LlamaDecoder.prefill_cached (task 1), which loads
    the prefix's blocks from the pool, prefills the 64 new tokens at pos0 = prefix and caches nothing new.  Host wall
    clock around the synchronous calls, median (min-max) of --reps alternating runs, each with fresh new tokens.
  - the load of the prefix's blocks: the k_kv_block_copy launch and one cudaMemcpyAsync per (block, layer, tensor) range,
    timed with CUDA events over --iters passes (zl_llama_kv_blocks_bench); bytes = what the copy reads plus writes, as a
    share of the H100 SXM data-sheet 3.35 TB/s.

    python tools/prefix_cache_bench.py [--out FILE] [--reps 7] [--iters 20]
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

PREFIXES = (512, 2048, 4096)
NEW = 64
BT = 128
PEAK = 3.35e12


def med(xs):
    return "%.2f (%.2f-%.2f)" % (statistics.median(xs), min(xs), max(xs))


def run(kv, reps, iters, log):
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    cfg = MODEL_PRESETS["llama-3.1-8b"]
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, max_batch=2, max_seq=max(PREFIXES) + 2 * NEW,
                       prefill_chunk=512, kv_cache_dtype=kv, **cfg)
    dec.init_synthetic(0)
    dec.enable_prefix_cache(sum(PREFIXES) // BT + 8, BT)
    rng = np.random.default_rng(0)
    V = cfg["vocab_size"]
    name = "int8 KV" if kv else "fp16 KV"
    goals = {}
    for P in PREFIXES:
        stem = rng.integers(0, V, P).astype(np.int32)
        new = lambda: np.concatenate([stem, rng.integers(0, V, NEW).astype(np.int32)])  # noqa: E731
        dec.prefill(0, new())                               # warm-up of every chunk shape
        _, c0 = dec.prefill_cached(1, new())                # fills the cache
        _, c1 = dec.prefill_cached(1, new())
        assert c0 == 0 and c1 == P, (c0, c1)
        cold, cached = [], []
        for _ in range(reps):
            p = new()
            t0 = time.perf_counter()
            dec.prefill(0, p)
            cold.append((time.perf_counter() - t0) * 1e3)
            p = new()
            t0 = time.perf_counter()
            _, c = dec.prefill_cached(1, p)
            cached.append((time.perf_counter() - t0) * 1e3)
            assert c == P
        hit = dec.prefix_cache.match(new())
        nb = len(hit)
        k_ms, nbytes = dec.bench_kv_blocks(1, range(nb), hit, load=True, iters=iters)
        m_ms, _ = dec.bench_kv_blocks(1, range(nb), hit, load=True, per_range_memcpy=True, iters=max(2, iters // 4))
        s_ms, _ = dec.bench_kv_blocks(1, range(nb), hit, load=False, iters=iters)
        ratio = statistics.median(cached) / statistics.median(cold)
        share = nbytes / (k_ms * 1e-3) / PEAK
        ranges = nb * cfg["num_layers"] * (4 if kv else 2)
        log("%s prefix %4d + %d  TTFT ms cold %s  cached %s  cached/cold %.3f" % (name, P, NEW, med(cold), med(cached), ratio))
        log("      load %d blocks (%.1f MB read + written): kernel %.1f us = %.0f GB/s = %.2f of 3.35 TB/s | "
            "%d x cudaMemcpyAsync %.1f us (%.2fx the kernel) | save kernel %.1f us"
            % (nb, nbytes / 1e6, k_ms * 1e3, nbytes / (k_ms * 1e-3) / 1e9, share, ranges, m_ms * 1e3, m_ms / k_ms,
               s_ms * 1e3))
        if P >= 2048:
            goals.setdefault("load", []).append(share)
        if P == 4096:
            goals["ttft"] = ratio
    dec.close()
    return name, goals


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prefix_cache_bench needs a CUDA device: nothing here runs on the CPU")
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: " + card())
    log("## Llama-3.1-8B GPTQ-int4 (synthetic, sym), prefill_chunk 512, %d-token blocks; shared prefix + %d new tokens. "
        "TTFT: host wall clock around the synchronous call, median (min-max) of %d alternating runs; copies: CUDA events "
        "over %d passes" % (BT, NEW, args.reps, args.iters))
    res = [run(kv, args.reps, args.iters, log) for kv in (None, "int8")]
    log("## goals (set before measuring)")
    for name, g in res:
        lo = min(g["load"])
        log("%s: load >= 0.6 of 3.35 TB/s at 2048+ tokens: %s (lowest %.2f);  cached TTFT at 4096 + 64 <= 0.1 of cold: %s "
            "(%.3f)" % (name, "met" if lo >= 0.6 else "missed", lo, "met" if g["ttft"] <= 0.1 else "missed", g["ttft"]))
    log_path = os.path.join(ROOT, "zhilight_b200", "build", "kv_pool.o.log")
    if os.path.exists(log_path):
        log("## ptxas -v, k_kv_block_copy (256 threads)")
        for ln in open(log_path).read().splitlines():
            if "k_kv_block_copy" in ln or ("registers" in ln or "spill" in ln):
                log(ln.strip())
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
