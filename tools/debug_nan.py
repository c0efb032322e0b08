#!/usr/bin/env python
"""Debug probe: decode the synthetic Llama-3.1-8B step by step through the host API and report the first step whose logits
are not finite (or whose picked token is invalid), for a few configuration variants."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(layers, steps, fuse, graph, pdl, batch):
    import torch
    from zhilight_b200.llama import LlamaDecoder, MODEL_PRESETS
    cfg = dict(MODEL_PRESETS["llama-3.1-8b"])
    cfg["num_layers"] = layers
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, max_batch=batch, max_seq=steps + 8, fuse=fuse, use_graph=graph,
                       use_pdl=pdl, **cfg)
    dec.init_synthetic(seed=1)
    rng = np.random.default_rng(0)
    tok = rng.integers(0, cfg["vocab_size"], size=batch).astype(np.int32)
    pos = np.zeros(batch, np.int32)
    first_bad = None
    stats = []
    for s in range(steps):
        nxt, logits = dec.decode(tok, pos, want_logits=True)
        fin = bool(np.isfinite(logits).all())
        if s in (0, 1, 31, 32, 33, 63, 64, 65, 127, 128, 129) or not fin:
            stats.append((s, fin, float(np.nanmax(np.abs(logits))) if np.isfinite(logits).any() else float("nan"), int(nxt[0])))
        if not fin or (nxt < 0).any() or (nxt >= cfg["vocab_size"]).any():
            first_bad = s
            break
        tok = rng.integers(0, cfg["vocab_size"], size=batch).astype(np.int32)   # prompt-like: fresh random tokens
        pos += 1
    dec.close()
    print("layers=%d fuse=%d graph=%d pdl=%d batch=%d env=%s -> first_bad=%s %s" % (
        layers, fuse, graph, pdl, batch, {k: v for k, v in os.environ.items() if k.startswith("ZL_")}, first_bad, stats), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1:
        a = [int(x) for x in sys.argv[1:7]]
        run(*a)
        sys.exit(0)
    variants = [({}, (32, 140, 2, 1, 1, 1)), ({}, (32, 140, 0, 1, 1, 1)), ({}, (32, 140, 2, 0, 0, 1)),
                ({}, (4, 140, 2, 1, 1, 1)), ({}, (32, 40, 2, 1, 1, 32))]
    for env, args in variants:
        e = dict(os.environ)
        e.update(env)
        subprocess.run([sys.executable, os.path.abspath(__file__)] + [str(x) for x in args], env=e, timeout=600)
