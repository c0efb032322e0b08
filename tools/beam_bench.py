"""Beam search on the decode driver: zl_beam_topk against zl_argmax, and 8B beam steps against decode steps.

    python tools/beam_bench.py [--out profiles/beam_bench.txt]

(1) selection: zl_beam_topk (groups of width min(R, 16), K = min(2 width, 32)) and zl_argmax on the same (R, 128256) fp32
    logits, CUDA events over 200 launches each, bytes read (R V 4) as a share of 3.35 TB/s;
(2) Llama-3.1-8B GPTQ-int4 synthetic weights, a 128-token prompt and 256 new tokens per group: beam_search per step
    (forward + pick, forks, host policy) and the beam step against the decode step at the same B, alternating, medians.
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from zhilight_b200 import _lib, ops  # noqa: E402
from zhilight_b200.llama import LlamaDecoder, MODEL_PRESETS, QUANT_GPTQ  # noqa: E402

HBM = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


def events_us(fn, n=200):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def selection(lines):
    V = 128256
    dev = torch.device("cuda:0")
    lines.append("(1) selection over (R, %d) fp32 logits, 200 launches each, CUDA events" % V)
    lines.append("  R   width  K   topk_us  argmax_us  ratio  topk_share_of_3.35TB/s")
    for R in (1, 4, 16, 32, 64):
        w = min(R, 16)
        k = min(2 * w, 32)
        g = np.array([[i * w, w] for i in range(R // w)], np.int32)
        x = torch.randn(R, V, device=dev) * 3
        cum = torch.zeros(R, device=dev)
        out = torch.empty(R, dtype=torch.int32, device=dev)
        parent = torch.empty(len(g), k, dtype=torch.int32, device=dev)
        token, score = torch.empty_like(parent), torch.empty(len(g), k, device=dev)
        nb = _lib.load().zl_beam_topk_workspace_bytes(R, V, k)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        anb = _lib.load().zl_argmax_workspace_bytes(R)
        aws = torch.empty(anb, dtype=torch.uint8, device=dev)
        gp = g.ctypes.data_as(__import__("ctypes").c_void_p)
        topk = lambda: _lib.call("zl_beam_topk", ops._p(x), R, V, ops._p(cum), gp, len(g), k, ops._p(parent),
                                 ops._p(token), ops._p(score), ops._p(ws), nb, 0, ops._stream())
        am = lambda: _lib.call("zl_argmax", ops._p(x), ops._p(out), R, V, ops._p(aws), anb, 0, ops._stream())
        t_k, t_a = [], []
        for _ in range(3):   # alternating rounds
            t_k.append(events_us(topk))
            t_a.append(events_us(am))
        tk, ta = float(np.median(t_k)), float(np.median(t_a))
        share = R * V * 4 / (tk * 1e-6) / HBM
        lines.append("  %-3d %-6d %-3d %8.2f %9.2f %6.2f  %.2f" % (R, w, k, tk, ta, tk / ta, share))
        yield R, tk, ta, share


def model_runs(lines, steps):
    cfg = MODEL_PRESETS["llama-3.1-8b"]
    prompt_len = 128
    dec = LlamaDecoder(quant_type=QUANT_GPTQ, max_batch=32, max_seq=prompt_len + steps + 8, prefill_chunk=128, **cfg)
    dec.init_synthetic(0)
    rng = np.random.default_rng(0)
    row_bytes = cfg["num_kv_heads"] * cfg["dim_head"] * 2
    stream = torch.cuda.ExternalStream(dec.stream())
    lines.append("(2) Llama-3.1-8B GPTQ-int4 synthetic, fp16 KV, %d-token prompt, %d new tokens (no EOS)"
                 % (prompt_len, steps))
    lines.append("  W  G  B   search_ms/step  beam_step_ms  decode_ms  beam/decode  search/decode  fork_MB/step  "
                 "fork_GB/s  host_policy_ms/step")
    out = {}
    for G in (1, 4):
        for W in (1, 2, 4, 8):
            B = W * G
            prompts = [list(rng.integers(0, cfg["vocab_size"], prompt_len)) for _ in range(G)]
            t_step, t_copy, copy_bytes, copy_ms = [0.0], [0.0], [0.0], []

            def step(t, p, g, c, k):
                t0 = time.perf_counter()
                r = dec.beam_step(t, p, g, c, k)
                t_step[0] += time.perf_counter() - t0
                return r

            def copy(ranges):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record(stream)
                dec.kv_copy_rows(ranges)
                e1.record(stream)
                t_copy[0] += time.perf_counter() - t0
                e1.synchronize()
                copy_ms.append(e0.elapsed_time(e1))
                copy_bytes[0] += float(sum(r[3] - r[2] for r in ranges)) * row_bytes * 2 * cfg["num_layers"]

            t_pf = [0.0]

            def prefill(s, toks):   # timed apart: not a step
                t0 = time.perf_counter()
                dec.prefill(s, np.array(toks, np.int32))
                t_pf[0] += time.perf_counter() - t0

            from zhilight_b200 import beam_search as bs
            trace = []
            t0 = time.perf_counter()
            bs.beam_search(step, copy, prefill, prompts, W, steps, -1, 1, trace)
            total = time.perf_counter() - t0 - t_pf[0]
            n = len(trace)
            # the beam step and the decode step at the same B and positions, alternating
            tok = np.zeros(B, np.int32)
            pos = np.full(B, prompt_len + steps // 2, np.int32)
            groups = np.array([[g * W, W] for g in range(G)], np.int32)
            cum = np.zeros(B, np.float32)
            k = min(2 * W, 32)
            tb, td = [], []
            for _ in range(30):
                a = time.perf_counter()
                dec.beam_step(tok, pos, groups, cum, k)
                b = time.perf_counter()
                dec.decode(tok, pos)
                c = time.perf_counter()
                tb.append(b - a)
                td.append(c - b)
            mb, md = np.median(tb) * 1e3, np.median(td) * 1e3
            per = total / n * 1e3
            policy = (total - t_step[0] - t_copy[0] - sum(copy_ms) * 1e-3) / n * 1e3
            rate = copy_bytes[0] * 2 / (sum(copy_ms) * 1e-3) / 1e9 if copy_ms else 0.0   # read + write
            lines.append("  %-2d %-2d %-3d %14.3f %13.3f %10.3f %12.3f %14.3f %13.2f %10.1f %19.3f"
                         % (W, G, B, per, mb, md, mb / md, per / md, copy_bytes[0] / n / 1e6, rate, policy))
            out[(W, G)] = (per, mb, md)
    dec.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=256)
    a = ap.parse_args()
    name, pl = card()
    lines = ["beam search bench: %s, power limit %s" % (name, pl)]
    sel = list(selection(lines))
    runs = model_runs(lines, a.steps)
    lines.append("goals:")
    worst = max(tk / ta for _, tk, ta, _ in sel)
    lines.append("  selection <= 1.5x zl_argmax time: worst %.2fx -> %s" % (worst, "met" if worst <= 1.5 else "not met"))
    big = min(s for r, _, _, s in sel if r >= 32)
    lines.append("  >= 0.5 of 3.35 TB/s at R >= 32: lowest %.2f -> %s" % (big, "met" if big >= 0.5 else "not met"))
    per, mb, md = runs[(4, 1)]
    lines.append("  8B W=4 G=1 search step <= 1.10x decode step: %.3f -> %s"
                 % (per / md, "met" if per / md <= 1.10 else "not met"))
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
