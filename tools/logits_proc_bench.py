"""Logits processors' cost: zl_sample with and without 300 logit-bias entries per row, k_ngram_levels' kernel time on
text-like and constant sequences, and Llama-3.1-8B GPTQ-int4 synthetic decode tok/s with every task's n-gram penalty and
bias against the same sampling without them (alternating runs in one process).

    python tools/logits_proc_bench.py [--out FILE] [--reps 5] [--steps 512]
"""
import argparse
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.sample_bench import card, ctypes_stream, time_us  # noqa: E402

SAMPLED = dict(temperature=0.8, top_p=0.95, repetition_penalty=1.1)


def _text_like(rng, n, V):
    """Zipf-distributed token ids: a few frequent tokens, a long tail, few long repeats"""
    import numpy as np
    return (np.minimum(rng.zipf(1.2, size=n), V) - 1).astype(np.int32)


def _state(dev, B, V, seqs, n_bias, rng):
    import numpy as np
    import torch
    stride = max(len(s) for s in seqs) + 8
    seq = np.zeros((B, stride), np.int32)
    for t, s in enumerate(seqs):
        seq[t, :len(s)] = s
    bt = np.stack([rng.choice(V, size=max(n_bias, 1), replace=False) for _ in range(B)]).astype(np.int32)
    bv = rng.uniform(-2, 2, size=bt.shape).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return dict(seq=t(seq), seq_len=t(np.array([len(s) for s in seqs], np.int32)), stride=stride, bias_tok=t(bt),
                bias_val=t(bv), bias_cnt=t(np.full(B, n_bias, np.int32)), bias_stride=bt.shape[1])


def _call_processed(lib, ops, _lib, logits, B, V, dparams, counter, out, st, ngram, ws, nb, s_ptr):
    base_len = st["seq_len"].clone()

    def run():
        st["seq_len"].copy_(base_len)   # every launch sees the same sequence length
        _lib.call("zl_sample_processed", ops._p(logits), B, V, ops._p(dparams), None, ops._p(counter), None, 0,
                  ops._p(ngram) if ngram is not None else None, ops._p(st["seq"]), ops._p(st["seq_len"]), st["stride"],
                  ops._p(st["bias_tok"]), ops._p(st["bias_val"]), ops._p(st["bias_cnt"]), st["bias_stride"], ops._p(out),
                  ops._p(ws) if ws is not None else None, nb, 0, s_ptr)
    return run


def bias_cost(log, V=128256, iters=300):
    import numpy as np
    import torch
    from zhilight_b200 import _lib, ops
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream()
    s_ptr = ctypes_stream(stream)
    rng = np.random.default_rng(0)
    log("## bias cost: us per call (CUDA events over %d calls), V = %d, 300 bias entries per row, no sequence" % (iters, V))
    log("%-24s %4s %10s %14s %8s" % ("setting", "B", "zl_sample", "+300 bias", "ratio"))
    for B in (1, 32):
        g = torch.Generator(device=dev).manual_seed(B)
        logits = torch.randn(B, V, device=dev, generator=g) * 3
        out = torch.empty(B, dtype=torch.int32, device=dev)
        counter = torch.arange(B, dtype=torch.int32, device=dev)
        st = _state(dev, B, V, [[1, 2, 3]] * B, 300, rng)
        for name, p in (("greedy", dict(temperature=0.0)), ("T0.8 top_p0.95", dict(temperature=0.8, top_p=0.95))):
            arr = ops.sample_params_array([dict(p, seed=i) for i in range(B)], B)
            dparams = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev)
            t0 = time_us(lambda: _lib.call("zl_sample", ops._p(logits), B, V, ops._p(dparams), None, ops._p(counter),
                                           None, 0, ops._p(out), None, 0, 0, s_ptr), iters, stream)
            t1 = time_us(lambda: _lib.call("zl_sample_processed", ops._p(logits), B, V, ops._p(dparams), None,
                                           ops._p(counter), None, 0, None, None, None, 0, ops._p(st["bias_tok"]),
                                           ops._p(st["bias_val"]), ops._p(st["bias_cnt"]), st["bias_stride"],
                                           ops._p(out), None, 0, 0, s_ptr), iters, stream)
            log("%-24s %4d %10.2f %14.2f %8.3f" % (name, B, t0, t1, t1 / t0))


def ngram_kernel(log, V=128256, iters=100):
    """k_ngram_levels' device time from torch.profiler (a run of its own, kernels named)"""
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from zhilight_b200 import _lib, ops
    lib = _lib.load()
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream()
    s_ptr = ctypes_stream(stream)
    rng = np.random.default_rng(1)
    log("## k_ngram_levels: us per launch (torch.profiler device time, mean of %d launches)" % iters)
    log("%-12s %6s %4s %10s %12s" % ("sequence", "n", "B", "k_ngram", "k_sample"))
    for kind in ("text", "constant"):
        for n in (1024, 4096):
            for B in (1, 8, 32):
                seqs = [_text_like(rng, n, V).tolist() if kind == "text" else [7] * n for _ in range(B)]
                st = _state(dev, B, V, seqs, 0, rng)
                g = torch.Generator(device=dev).manual_seed(B)
                logits = torch.randn(B, V, device=dev, generator=g) * 3
                out = torch.empty(B, dtype=torch.int32, device=dev)
                counter = torch.arange(B, dtype=torch.int32, device=dev)
                arr = ops.sample_params_array([dict(SAMPLED, seed=i) for i in range(B)], B)
                dparams = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev)
                ngram = torch.full((B,), 1.1, dtype=torch.float32, device=dev)
                nb = lib.zl_sample_processed_workspace_bytes(B, st["stride"])
                ws = torch.empty(nb, dtype=torch.uint8, device=dev)
                run = _call_processed(lib, ops, _lib, logits, B, V, dparams, counter, out, st, ngram, ws, nb, s_ptr)
                for _ in range(10):
                    run()
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(iters):
                        run()
                    torch.cuda.synchronize()
                t = {}
                for e in prof.key_averages():
                    dt = getattr(e, "device_time_total", None)
                    if dt is None:
                        dt = e.cuda_time_total
                    for k in ("k_ngram_levels", "k_sample"):
                        if k in e.key:
                            t[k] = t.get(k, 0.0) + dt / iters
                log("%-12s %6d %4d %10.2f %12.2f" % (kind, n, B, t.get("k_ngram_levels", float("nan")),
                                                     t.get("k_sample", float("nan"))))


def decode_rates(log, reps, steps, warm=8):
    import numpy as np
    import torch
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    cfg = dict(MODEL_PRESETS["llama-3.1-8b"])
    V = cfg["vocab_size"]
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, dtype="f16", max_batch=32, max_seq=1024, **cfg)
    dec.init_synthetic(seed=1)
    stream = torch.cuda.ExternalStream(dec.stream())
    rng = np.random.default_rng(0)
    biases = [{int(k): float(v) for k, v in zip(rng.choice(V, 50, replace=False), rng.uniform(-2, 2, 50))}
              for _ in range(32)]
    log("## Llama-3.1-8B GPTQ-int4 (synthetic weights) decode, device-resident steps, %d generated tokens per run (the "
        "sequence is cleared before each run), %d alternating runs per mode" % (steps, reps))
    log("plain = %s for every task; processors = the same plus ngram_penalty 1.1 and 50 logit_bias entries" % SAMPLED)
    for B in (1, 32):
        tok = rng.integers(0, V, size=B).astype(np.int32)
        pos = np.full(B, 128, dtype=np.int32)
        res = {"plain": [], "processors": []}
        for _ in range(reps):
            for mode in ("plain", "processors"):
                for t in range(B):
                    if mode == "plain":
                        dec.set_sampling(t, seed=t, **SAMPLED)
                    else:
                        dec.set_sampling(t, seed=t, ngram_penalty=1.1, logit_bias=biases[t], **SAMPLED)
                dec.set_state(tok, pos)
                for _ in range(warm):   # warms the graph; the sequence then holds `warm` tokens
                    dec.step_device(B)
                dec.sync()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(steps):
                    dec.step_device(B)
                e1.record(stream)
                e1.synchronize()
                res[mode].append(B * steps * 1000.0 / e0.elapsed_time(e1))
        a, b = statistics.median(res["plain"]), statistics.median(res["processors"])
        log("B=%-3d plain %.1f tok/s (%.1f-%.1f)  processors %.1f tok/s (%.1f-%.1f)  processors/plain %.4f" % (
            B, a, min(res["plain"]), max(res["plain"]), b, min(res["processors"]), max(res["processors"]), b / a))
    dec.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=512)
    ap.add_argument("--no-decode", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("logits_proc_bench needs a CUDA device")
    from zhilight_b200 import build
    build.build()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: %s" % card())
    bias_cost(log)
    ngram_kernel(log)
    if not args.no_decode:
        decode_rates(log, args.reps, args.steps)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
