"""Sampler cost: zl_sample kernel time against zl_argmax, and Llama-3.1-8B GPTQ-int4 synthetic decode tok/s with every
task greedy against every task sampled (alternating runs in one process).

    python tools/sample_bench.py [--out FILE] [--reps 5] [--steps 128]
"""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SETTINGS = {
    "greedy": dict(temperature=0.0),
    "T0.8": dict(temperature=0.8),
    "T0.8 top_p0.95": dict(temperature=0.8, top_p=0.95),
    "T0.8 top_k50": dict(temperature=0.8, top_k=50),
    "T0.8 top_k50 top_p0.95": dict(temperature=0.8, top_k=50, top_p=0.95),
    "T0.8 top_k50 top_p0.95 rep1.1 pres0.2": dict(temperature=0.8, top_k=50, top_p=0.95, repetition_penalty=1.1,
                                                  presence_penalty=0.2),
}


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        q = "nvidia-smi unavailable (%s)" % e
    return "%s | %s" % (torch.cuda.get_device_name(0), q)


def time_us(fn, iters, stream):
    import torch
    for _ in range(10):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / iters


def kernel_times(log, V=128256, iters=200):
    import torch
    from zhilight_b200 import _lib, ops
    lib = _lib.load()
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream()
    log("## kernel time (us per launch, CUDA events over %d launches), V = %d" % (iters, V))
    log("%-40s %6s %10s %10s" % ("setting", "B", "zl_sample", "zl_argmax"))
    for B in (1, 8, 32, 128):
        g = torch.Generator(device=dev).manual_seed(B)
        logits = torch.randn(B, V, device=dev, generator=g) * 3
        out = torch.empty(B, dtype=torch.int32, device=dev)
        nb = lib.zl_argmax_workspace_bytes(B)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        s_ptr = ctypes_stream(stream)
        t_arg = time_us(lambda: _lib.call("zl_argmax", ops._p(logits), ops._p(out), B, V, ops._p(ws), nb, 0, s_ptr),
                        iters, stream)
        counter = torch.arange(B, dtype=torch.int32, device=dev)
        hist = torch.zeros(B, (V + 31) // 32, dtype=torch.int32, device=dev)
        hist[:, ::97] = 0x01010101
        for name, p in SETTINGS.items():
            arr = ops.sample_params_array([dict(p, seed=i) for i in range(B)], B)
            dparams = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev)
            pen = "repetition_penalty" in p
            h = ops._p(hist) if pen else None
            hw = hist.shape[1] if pen else 0
            t = time_us(lambda: _lib.call("zl_sample", ops._p(logits), B, V, ops._p(dparams), None, ops._p(counter), h, hw,
                                          ops._p(out), None, 0, 0, s_ptr), iters, stream)
            log("%-40s %6d %10.2f %10.2f" % (name, B, t, t_arg))


def ctypes_stream(stream):
    import ctypes
    return ctypes.c_void_p(stream.cuda_stream)


def decode_rates(log, reps, steps, warm=8):
    import numpy as np
    import torch
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    cfg = dict(MODEL_PRESETS["llama-3.1-8b"])
    cfg.pop("qkv_bias", None)
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, dtype="f16", max_batch=32, max_seq=512, **cfg)
    dec.init_synthetic(seed=1)
    stream = torch.cuda.ExternalStream(dec.stream())
    sampled = SETTINGS["T0.8 top_k50 top_p0.95 rep1.1 pres0.2"]
    log("## Llama-3.1-8B GPTQ-int4 (synthetic weights) decode, device-resident steps, %d timed steps per run, "
        "%d alternating runs per mode" % (steps, reps))
    log("sampled = %s for every task" % sampled)
    rng = np.random.default_rng(0)
    for B in (1, 32):
        tok = rng.integers(0, cfg["vocab_size"], size=B).astype(np.int32)
        pos = np.full(B, 128, dtype=np.int32)
        res = {"greedy": [], "sampled": []}
        for _ in range(reps):
            for mode in ("greedy", "sampled"):
                for t in range(B):
                    if mode == "greedy":
                        dec.set_sampling(t)
                    else:
                        dec.set_sampling(t, seed=t, **sampled)
                dec.set_state(tok, pos)
                for _ in range(warm):
                    dec.step_device(B)
                dec.sync()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(steps):
                    dec.step_device(B)
                e1.record(stream)
                e1.synchronize()
                ms = e0.elapsed_time(e1)
                res[mode].append(B * steps * 1000.0 / ms)
        g, s = statistics.median(res["greedy"]), statistics.median(res["sampled"])
        log("B=%-3d greedy %.1f tok/s (%.1f-%.1f)  sampled %.1f tok/s (%.1f-%.1f)  sampled/greedy %.4f  "
            "(%.3f vs %.3f ms/step)" % (B, g, min(res["greedy"]), max(res["greedy"]), s, min(res["sampled"]),
                                        max(res["sampled"]), s / g, B * 1000.0 / g, B * 1000.0 / s))
    dec.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--no-decode", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench needs a CUDA device")
    from zhilight_b200 import build
    build.build()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: %s" % card())
    kernel_times(log)
    if not args.no_decode:
        decode_rates(log, args.reps, args.steps)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
