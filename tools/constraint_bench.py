"""Constrained decoding's cost: zl_sample_masked (every row masked to half the vocabulary) against zl_sample_processed
over the same rows, and Llama-3.1-8B GPTQ-int4 synthetic generate tok/s with every task constrained (a one-state mask, a
`choices` trie) against the same sampling unconstrained (alternating runs in one process), and a host loop of decode
steps that uploads a fresh one-state mask per step against generate.

    python tools/constraint_bench.py [--out FILE] [--reps 3] [--steps 128]
"""
import argparse
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.sample_bench import card, ctypes_stream, time_us  # noqa: E402

SAMPLED = dict(temperature=0.8, top_p=0.95)


def sampler_cost(log, V=128256, iters=300):
    import numpy as np
    import torch
    from zhilight_b200 import _lib, ops
    from zhilight_b200.constraints import token_bitmask
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream()
    s_ptr = ctypes_stream(stream)
    rng = np.random.default_rng(0)
    log("## sampler: us per call (CUDA events over %d calls), V = %d, every row masked to V/2 random tokens" % (iters, V))
    log("%-16s %4s %20s %18s %8s" % ("setting", "T", "zl_sample_processed", "zl_sample_masked", "ratio"))
    for name, p in (("greedy", dict(temperature=0.0)), ("T0.8 top_p0.95", SAMPLED)):
        for T in (1, 8, 32):
            g = torch.Generator(device=dev).manual_seed(T)
            logits = torch.randn(T, V, device=dev, generator=g) * 3
            out = torch.empty(T, dtype=torch.int32, device=dev)
            counter = torch.arange(T, dtype=torch.int32, device=dev)
            arr = ops.sample_params_array([dict(p, seed=i) for i in range(T)], T)
            dparams = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev)
            masks = np.stack([token_bitmask(rng.choice(V, V // 2, replace=False), V) for _ in range(T)])
            dmask = torch.from_numpy(masks.view(np.int32)).to(dev)
            W = masks.shape[1]
            t0 = time_us(lambda: _lib.call("zl_sample_processed", ops._p(logits), T, V, ops._p(dparams), None,
                                           ops._p(counter), None, 0, None, None, None, 0, None, None, None, 0,
                                           ops._p(out), None, 0, 0, s_ptr), iters, stream)
            t1 = time_us(lambda: _lib.call("zl_sample_masked", ops._p(logits), T, V, ops._p(dparams), None,
                                           ops._p(counter), None, 0, None, None, None, 0, None, None, None, 0,
                                           ops._p(dmask), W, None, ops._p(out), None, 0, 0, s_ptr), iters, stream)
            log("%-16s %4d %20.2f %18.2f %8.3f" % (name, T, t0, t1, t1 / t0))


def _trie(V, rng):
    from zhilight_b200.constraints import choices
    seqs = [rng.choice(np.arange(3, V), 32, replace=False).tolist() for _ in range(4)]
    return choices(seqs, [1, 2], V)


def _rate(dec, stream, B, tok, pos, steps, setup, run):
    import torch
    setup()
    dec.set_state(tok, pos)
    dec.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    run()
    e1.record(stream)
    e1.synchronize()
    return B * steps * 1000.0 / e0.elapsed_time(e1)


def generate_rates(log, reps, steps):
    import torch
    from zhilight_b200.constraints import allowed
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    cfg = dict(MODEL_PRESETS["llama-3.1-8b"])
    V = cfg["vocab_size"]
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, dtype="f16", max_batch=32, max_seq=512, **cfg)
    dec.init_synthetic(seed=1)
    rng = np.random.default_rng(0)
    trie = _trie(V, rng)
    dec.enable_constraints(trie.n_states, trie.n_edges)
    stream = torch.cuda.ExternalStream(dec.stream())
    half = allowed(rng.choice(V, V // 2, replace=False), V)
    step_masks = [allowed(rng.choice(V, V // 2, replace=False), V) for _ in range(8)]
    log("## Llama-3.1-8B GPTQ-int4 (synthetic weights) generate, %d steps per run from position 128, no stop ids, "
        "%d alternating runs per mode; every task samples with %s" % (steps, reps, SAMPLED))
    log("unconstrained: no automaton; mask: a one-state automaton allowing V/2 random tokens; trie: choices() over 4 "
        "sequences of 32 tokens (%d states), then its final state; host-mask: decode() steps, each after a fresh "
        "one-state V/2 mask per task" % trie.n_states)
    for B in (1, 8, 32):
        tok = rng.integers(0, V, size=B).astype(np.int32)
        pos = np.full(B, 128, dtype=np.int32)
        positions = pos.copy()

        def arm(aut):
            def setup():
                for t in range(B):
                    dec.set_sampling(t, seed=t, **SAMPLED)
                    dec.set_constraint(t, aut)
                    dec.set_stop(t)
            return setup

        def gen():
            dec.generate(B, steps)

        def host():
            tk = tok.copy()
            for s in range(steps):
                for t in range(B):
                    dec.set_constraint(t, step_masks[s % len(step_masks)])
                tk = dec.decode(tk, positions + s)

        modes = {"unconstrained": (arm(None), gen), "mask": (arm(half), gen), "trie": (arm(trie), gen),
                 "host-mask": (arm(None), host)}
        for setup, run in modes.values():   # warms every graph
            _rate(dec, stream, B, tok, pos, steps, setup, run)
        res = {k: [] for k in modes}
        for _ in range(reps):
            for k, (setup, run) in modes.items():
                res[k].append(_rate(dec, stream, B, tok, pos, steps, setup, run))
        med = {k: statistics.median(v) for k, v in res.items()}
        log("B=%-3d " % B + "  ".join("%s %.1f tok/s (%.1f-%.1f)" % (k, med[k], min(res[k]), max(res[k])) for k in modes))
        log("      mask/unconstrained %.4f  trie/unconstrained %.4f (goal >= 0.98)  host-mask/mask %.4f" % (
            med["mask"] / med["unconstrained"], med["trie"] / med["unconstrained"], med["host-mask"] / med["mask"]))
    dec.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--no-generate", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("constraint_bench needs a CUDA device")
    from zhilight_b200 import build
    build.build()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: %s" % card())
    sampler_cost(log)
    if not args.no_generate:
        generate_rates(log, args.reps, args.steps)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
