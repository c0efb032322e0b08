"""Generate until stop: Llama-3.1-8B GPTQ-int4 (synthetic weights), 128-token prompts, 256 new tokens at B = 1 / 8 / 32.
Three modes, alternating runs, medians of wall time (host clock around work that ends in a sync) and tok/s of emitted
tokens:
  host     decode() in a host loop with the stop check in Python (one sync per step)
  device   step_device() x 256 with no stop rule (the upper bound: no stop check at all)
  generate one generate(b, 256) call
Then an early-stop scenario: half the tasks get, as their stop id, the token they emit at step 64 of a greedy reference
pass; host loop against generate.  Prints the card and its power limit.

    python tools/generate_bench.py [--out FILE] [--reps 5]
"""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.sample_bench import card  # noqa: E402

PROMPT, NEW, MAX_BATCH = 128, 256, 32


def _host(dec, b, tok0, stops):
    """decode() steps with the stop check on the host; a finished row is fed its frozen state.  -> emitted tokens"""
    import numpy as np
    tok, pos = tok0.copy(), np.full(b, PROMPT, np.int32)
    live = np.ones(b, bool)
    n = 0
    for _ in range(NEW):
        nxt = dec.decode(tok, pos)
        for t in np.nonzero(live)[0]:
            n += 1
            if int(nxt[t]) in stops[t]:
                live[t] = False
            tok[t] = nxt[t]
            pos[t] += 1
        if not live.any():
            break
    return n


def _device(dec, b, tok0, stops):
    import numpy as np
    dec.set_state(tok0, np.full(b, PROMPT, np.int32))
    for _ in range(NEW):
        dec.step_device(b)
    dec.sync()
    return b * NEW


def _generate(dec, b, tok0, stops):
    import numpy as np
    for t in range(b):
        dec.set_stop(t, stops[t])
    dec.set_state(tok0, np.full(b, PROMPT, np.int32))
    out, _, _ = dec.generate(b, NEW)
    return sum(o.size for o in out)


MODES = {"host": _host, "device": _device, "generate": _generate}


def _run(log, dec, b, tok0, stops, modes, reps):
    res = {m: [] for m in modes}
    for m in modes:   # warm-up: graphs of every bucket
        MODES[m](dec, b, tok0, stops)
    for _ in range(reps):
        for m in modes:
            t0 = time.perf_counter()
            n = MODES[m](dec, b, tok0, stops)
            dt = time.perf_counter() - t0
            res[m].append((dt, n))
    row = []
    med = {}
    for m in modes:
        dts = [d for d, _ in res[m]]
        n = res[m][0][1]
        med[m] = n / statistics.median(dts)
        row.append("%s %.1f ms %.1f tok/s (%d tokens; %.1f-%.1f)" % (
            m, 1000 * statistics.median(dts), med[m], n, n / max(dts), n / min(dts)))
    log("B=%-3d " % b + " | ".join(row))
    return med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("generate_bench needs a CUDA device")
    from zhilight_b200 import build
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    build.build()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: %s" % card())
    cfg = dict(MODEL_PRESETS["llama-3.1-8b"])
    V = cfg["vocab_size"]
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, dtype="f16", max_batch=MAX_BATCH, max_seq=512,
                       prefill_chunk=PROMPT, **cfg)
    dec.init_synthetic(seed=1)
    rng = np.random.default_rng(0)
    first = np.array([dec.prefill(t, rng.integers(0, V, PROMPT).astype(np.int32)) for t in range(MAX_BATCH)], np.int32)
    log("## Llama-3.1-8B GPTQ-int4 (synthetic weights), greedy, %d-token prompts, %d new tokens, %d alternating runs "
        "per mode, medians (min-max tok/s)" % (PROMPT, NEW, args.reps))
    ratios = []
    for b in (1, 8, 32):
        med = _run(log, dec, b, first[:b].copy(), [()] * b, ("host", "device", "generate"), args.reps)
        ratios.append((b, med["generate"] / med["device"], med["generate"] / med["host"]))
    for b, rd, rh in ratios:
        log("B=%-3d generate / device %.4f (goal >= 0.99)  generate / host %.4f (goal at B=1: >= 1.04)" % (b, rd, rh))
    log("## early stop: tasks 0, 2, 4, ... stop at the token they emit at step 64 of a greedy pass; the others run %d "
        "steps" % NEW)
    for b in (1, 8, 32):
        dec.set_state(first[:b], np.full(b, PROMPT, np.int32))
        for t in range(b):
            dec.set_stop(t)
        ref, _, _ = dec.generate(b, NEW)
        stops = [(int(ref[t][64]),) if t % 2 == 0 else () for t in range(b)]
        med = _run(log, dec, b, first[:b].copy(), stops, ("host", "generate"), args.reps)
        log("B=%-3d generate / host %.4f" % (b, med["generate"] / med["host"]))
    dec.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
