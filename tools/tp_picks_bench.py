"""Full-vocabulary picks under tensor parallelism (LlamaDecoder.enable_tp_picks).  Run one process per GPU:

    python -m torch.distributed.run --nproc_per_node 2 tools/tp_picks_bench.py [--out FILE] [--reps 5]

1. The vocabulary all-gather kernel (zl_vocab_allgather) at T = 1 / 8 / 32 rows of V = 128256, by CUDA events over
   back-to-back launches replayed from a CUDA graph: the bytes each rank sends, T * vshard * 4 * (ws - 1), over that
   time, and their share of the 450 GB/s per direction of NVLink in the H100 SXM data sheet.
2. Llama-3.1-8B GPTQ-int4 (synthetic weights) at TP = ws, 128-token prompts, B = 1 / 8 / 32, decode tok/s in medians of
   alternating runs of 128 steps: greedy on a decoder without the gather (the candidate exchange), greedy with picks
   enabled, and sampled (T 0.8, top-k 50, top-p 0.95) through a step_device loop, decode() and generate().
Rank 0 prints the card and its power limit and writes the report.
"""
import argparse
import ctypes
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.sample_bench import card  # noqa: E402

PROMPT, STEPS, MAX_BATCH, V = 128, 128, 32, 128256
NVLINK_GBS = 450.0
SAMPLED = dict(temperature=0.8, top_k=50, top_p=0.95)


def _gather_times(log, rank, ws, dev, iters=200):
    import torch
    import torch.distributed as dist
    from zhilight_b200.dist import VocabGather
    g = VocabGather(MAX_BATCH, V, rank, ws)
    vs = V // ws
    log("## zl_vocab_allgather, V = %d, ws = %d, %d back-to-back launches per size replayed from a CUDA graph"
        % (V, ws, iters))
    for T in (1, 8, 32):
        shard = torch.randn((T, vs), dtype=torch.float32, device=dev)
        for _ in range(20):
            g.gather(shard)
        torch.cuda.synchronize()
        # the launches replay from a CUDA graph, so that the host does not pace them
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            for _ in range(iters):
                g.lib.zl_vocab_allgather(g.handle, ctypes.c_void_p(shard.data_ptr()), T, vs, 0, s)
        graph.replay()
        torch.cuda.synchronize()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        us = 1000.0 * e0.elapsed_time(e1) / iters
        sent = T * vs * 4 * (ws - 1)
        gbs = sent / us / 1e3
        log("T=%-3d %.2f us per gather, %d bytes sent per rank, %.1f GB/s = %.1f %% of %.0f GB/s" % (
            T, us, sent, gbs, 100.0 * gbs / NVLINK_GBS, NVLINK_GBS))
    dist.barrier()
    g.close()


def _device_loop(dec, b, tok0):
    import numpy as np
    dec.set_state(tok0, np.full(b, PROMPT, np.int32))
    for _ in range(STEPS):
        dec.step_device(b)
    dec.sync()


def _decode_loop(dec, b, tok0):
    import numpy as np
    tok, pos = tok0.copy(), np.full(b, PROMPT, np.int32)
    for _ in range(STEPS):
        tok = dec.decode(tok, pos)
        pos = pos + 1


def _generate(dec, b, tok0):
    import numpy as np
    for t in range(b):
        dec.set_stop(t)
    dec.set_state(tok0, np.full(b, PROMPT, np.int32))
    dec.generate(b, STEPS)


def _sampling(dec, b, on):
    for t in range(b):
        dec.set_sampling(t, **(dict(SAMPLED, seed=t) if on else {}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        raise SystemExit("tp_picks_bench needs CUDA devices")
    rank, ws = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=ws)
    from zhilight_b200 import build
    from zhilight_b200 import dist as zdist
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    build.build()
    lines = []

    def log(s):
        if rank == 0:
            print(s, flush=True)
            lines.append(s)

    log("card: %s" % card())
    _gather_times(log, rank, ws, dev)

    cfg = dict(MODEL_PRESETS["llama-3.1-8b"])
    decs = {}
    comms = []
    for name in ("plain", "picks"):
        d = LlamaDecoder(quant_type=5, group_size=128, sym=True, dtype="f16", max_batch=MAX_BATCH, max_seq=512,
                         prefill_chunk=PROMPT, tp_rank=rank, tp_size=ws, **cfg)
        if ws > 1:
            c = zdist.TPComm(PROMPT * cfg["dim_model"], rank, ws)
            d.set_comm(c)
            comms.append(c)
        d.init_synthetic(seed=1)
        if name == "picks":
            d.enable_tp_picks()
        decs[name] = d
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, V, PROMPT).astype(np.int32) for _ in range(MAX_BATCH)]
    first = {n: np.array([d.prefill(t, p) for t, p in enumerate(prompts)], np.int32) for n, d in decs.items()}
    modes = {
        "greedy (no gather)": (decs["plain"], False, _device_loop),
        "greedy (picks on)": (decs["picks"], False, _device_loop),
        "sampled step_device": (decs["picks"], True, _device_loop),
        "sampled decode": (decs["picks"], True, _decode_loop),
        "sampled generate": (decs["picks"], True, _generate),
    }
    log("## Llama-3.1-8B GPTQ-int4 (synthetic weights), TP=%d, %d-token prompts, %d steps, %d alternating runs per "
        "mode, medians (min-max tok/s); sampled = %s" % (ws, PROMPT, STEPS, args.reps, SAMPLED))
    for b in (1, 8, 32):
        res = {m: [] for m in modes}
        for rep in range(args.reps + 1):   # run 0 warms up every graph
            for m, (d, samp, fn) in modes.items():
                _sampling(d, b, samp)
                dist.barrier()
                t0 = time.perf_counter()
                fn(d, b, first["plain" if d is decs["plain"] else "picks"][:b].copy())
                dt = time.perf_counter() - t0
                if rep:
                    res[m].append(b * STEPS / dt)
        med = {m: statistics.median(v) for m, v in res.items()}
        log("B=%-3d " % b + " | ".join("%s %.1f (%.1f-%.1f)" % (m, med[m], min(res[m]), max(res[m])) for m in modes))
        g0 = med["greedy (no gather)"]
        log("B=%-3d sampled step_device / greedy %.4f (goal >= 0.95 at B = 8, 32)  greedy picks on / off %.4f (goal >= "
            "0.99)  generate / step_device %.4f (goal >= 0.99)  decode / greedy %.4f" % (
                b, med["sampled step_device"] / g0, med["greedy (picks on)"] / g0,
                med["sampled generate"] / med["sampled step_device"], med["sampled decode"] / g0))
    for d in decs.values():
        d.close()
    for c in comms:
        c.close()
    if args.out and rank == 0:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
