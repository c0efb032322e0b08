"""KV arena (kv_rows > 0) against the fixed layout, Llama-3.1-8B GPTQ-int4 (synthetic weights).  Prints the card and its
power limit, then:
  decode    step_device tok/s at B = 1 / 8 / 32 (context 512) with kv_rows = max_batch * max_seq against kv_rows = 0,
            alternating runs, medians
  relocate  k_kv_relocate moving one task of 512 / 2048 / 8192 rows over 32 layers, K and V (fp16, 8 kv heads x 128):
            read + write bytes over event time
  generate  B = 32, 128-token prompts, generate(32, 1024) from tasks released to zero capacity (the grants happen inside
            the timed call) against the fixed layout
  compact   the latency of a compaction inside a call: 32 tasks of 128 rows fill a 4160-row arena, task 0 is released
            and task 15 writes its row 128, which makes 14 tasks slide down and 16 slide up in pieces; the 1-token
            prefill that triggers it against the same prefill once the rows are granted (moves and launches from
            zl_kv_arena_replay of the same calls)
  capacity  max_seq 32768: 64 tasks of 128-token prompts generating 512 tokens each in an arena sized to their rows,
            against the largest B the fixed layout can allocate at that max_seq (searched down from the B whose KV
            alone exceeds the free memory, so B + 1 was tried and failed)

    python tools/kv_arena_bench.py [--out FILE] [--reps 5] [--skip-capacity]
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

MAX_BATCH, MAX_SEQ, CTX = 32, 2048, 512


def _model(kv_rows, max_batch=MAX_BATCH, max_seq=MAX_SEQ):
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    cfg = dict(MODEL_PRESETS["llama-3.1-8b"])
    dec = LlamaDecoder(quant_type=5, dtype="f16", max_batch=max_batch, max_seq=max_seq, prefill_chunk=512, sym=True,
                       kv_rows=kv_rows, **cfg)
    try:
        dec.init_synthetic(seed=1)
    except Exception:
        dec.close()
        raise
    return dec


def _decode_tps(dec, b, steps=64):
    import numpy as np
    dec.set_state(np.zeros(b, np.int32), np.full(b, CTX, np.int32))
    for _ in range(8):
        dec.step_device(b)
    dec.set_state(np.zeros(b, np.int32), np.full(b, CTX, np.int32))
    dec.sync()
    t0 = time.perf_counter()
    for _ in range(steps):
        dec.step_device(b)
    dec.sync()
    return b * steps / (time.perf_counter() - t0)


def _prompts(dec, b, n, vocab):
    import numpy as np
    rng = np.random.default_rng(0)
    return [dec.prefill(t, rng.integers(0, vocab, n).astype(np.int32)) for t in range(b)]


def _generate_tps(dec, b, prompt, new, vocab, release):
    import numpy as np
    if release:
        for t in range(b):
            dec.kv_release(t)
    first = _prompts(dec, b, prompt, vocab)
    if release:
        for t in range(b):   # zero capacity past the prompt: generate grants the rest inside the timed call
            assert dec.kv_capacity(t) < prompt + new
    for t in range(b):
        dec.set_stop(t, (), 0)
    dec.set_state(np.array(first, np.int32), np.full(b, prompt, np.int32))
    dec.sync()
    t0 = time.perf_counter()
    out, _, _ = dec.generate(b, new)
    dt = time.perf_counter() - t0
    return sum(o.size for o in out) / dt


def relocate_bw(lines, reps):
    import numpy as np
    import torch
    from zhilight_b200 import _lib
    layers, row = 32, 8 * 128 * 2
    for n in (512, 2048, 8192):
        rows = 2 * n
        bufs = [torch.empty(rows * row, dtype=torch.uint8, device="cuda") for _ in range(2 * layers)]
        bases = []
        for l in range(layers):
            bases += [bufs[2 * l].data_ptr(), bufs[2 * l + 1].data_ptr(), 0, 0]
        tab = torch.tensor(bases, dtype=torch.int64, device="cuda")
        mv = torch.tensor([[0, n, n, 0]], dtype=torch.int32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        lib = _lib.load()
        call = lambda: _lib.check(lib.zl_kv_relocate(ctypes.c_void_p(tab.data_ptr()), layers,
                                                     ctypes.c_void_p(mv.data_ptr()), 1, n, row, 0, ctypes.c_void_p(st)))
        for _ in range(3):
            call()
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                call()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / 10)
        t = statistics.median(ms)
        by = 2.0 * layers * 2 * n * row
        lines.append("relocate %5d rows x 32 layers K+V: %.3f ms  %.0f GB/s  %.2f of 3.35 TB/s"
                     % (n, t, by / t / 1e6, by / t / 1e6 / 3350))
        del bufs


def compaction_latency(lines, reps, vocab):
    import numpy as np
    from zhilight_b200.llama import kv_arena_replay
    tasks, prompt = 32, 128
    kv_rows = tasks * prompt + 64
    calls = [(t, prompt) for t in range(tasks)] + [(0, 0), (15, prompt + 1)]
    _, _, moves = kv_arena_replay(kv_rows, tasks, MAX_SEQ, calls)
    last = moves[moves[:, 0] == len(calls) - 1]
    n_launch = len(set(last[:, 1].tolist()))
    dec = _model(kv_rows)
    rng = np.random.default_rng(0)
    tok = rng.integers(0, vocab, (tasks, prompt)).astype(np.int32)
    with_c, without = [], []
    for _ in range(reps):
        for t in range(tasks):
            dec.kv_release(t)
        for t in range(tasks):
            dec.prefill(t, tok[t])
        dec.kv_release(0)
        dec.sync()
        t0 = time.perf_counter()
        dec.prefill(15, tok[15][:1], pos0=prompt)   # grants rows up to 129: the compaction
        with_c.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        dec.prefill(15, tok[15][:1], pos0=prompt)   # the rows are held now
        without.append(time.perf_counter() - t0)
    dec.close()
    mc, mw = statistics.median(with_c) * 1e3, statistics.median(without) * 1e3
    lines.append("compaction in a 1-token prefill (%d moves in %d k_kv_relocate launches): %.2f ms against %.2f ms without, "
                 "+%.2f ms" % (len(last), n_launch, mc, mw, mc - mw))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-capacity", action="store_true")
    args = ap.parse_args()
    import torch
    lines = [card()]
    vocab = 128256
    fixed, arena = _model(None), _model(MAX_BATCH * MAX_SEQ)
    for b in (1, 8, 32):
        f, a = [], []
        for _ in range(args.reps):
            f.append(_decode_tps(fixed, b))
            a.append(_decode_tps(arena, b))
        mf, ma = statistics.median(f), statistics.median(a)
        lines.append("decode B=%2d ctx %d: fixed %.1f tok/s  arena %.1f tok/s  ratio %.4f" % (b, CTX, mf, ma, ma / mf))
    f, a = [], []
    for _ in range(max(3, args.reps // 2)):
        f.append(_generate_tps(fixed, 32, 128, 1024, vocab, False))
        a.append(_generate_tps(arena, 32, 128, 1024, vocab, True))
    mf, ma = statistics.median(f), statistics.median(a)
    lines.append("generate B=32 prompt 128 new 1024: fixed %.1f tok/s  arena (grown in the call) %.1f tok/s  ratio %.4f"
                 % (mf, ma, ma / mf))
    fixed.close()
    arena.close()
    del fixed, arena
    relocate_bw(lines, args.reps)
    compaction_latency(lines, args.reps, vocab)
    if not args.skip_capacity:
        seq, tasks, prompt, new = 32768, 64, 128, 512
        kv_rows = tasks * 640
        dec = _model(kv_rows, max_batch=tasks, max_seq=seq)
        ta = _generate_tps(dec, tasks, prompt, new, vocab, False)
        dec.close()
        torch.cuda.empty_cache()
        lines.append("capacity max_seq %d: arena of %d rows (%.1f GiB fp16 KV), B=%d: %.1f tok/s"
                     % (seq, kv_rows, kv_rows * 131072 / 2**30, tasks, ta))
        need = tasks * seq * 131072 / 2**30
        # B + 1 tasks' KV alone exceeds the free memory, so the search starts above every B that can fit
        bound = int(torch.cuda.mem_get_info()[0] // (seq * 131072)) + 1
        b, failed = None, []
        for cand in range(bound, 0, -1):
            try:
                dec = _model(None, max_batch=cand, max_seq=seq)
            except Exception:
                failed.append(cand)
                torch.cuda.empty_cache()
                continue
            b = cand
            break
        if b is None:
            lines.append("capacity max_seq %d: the fixed layout allocates no B up to %d" % (seq, bound))
        else:
            tf = _generate_tps(dec, b, prompt, new, vocab, False)
            dec.close()
            lines.append("capacity max_seq %d: the fixed layout needs %.0f GiB of fp16 KV for B=%d; largest B it allocates: "
                         "%d (tried and failed: %s), %.1f tok/s (arena / fixed %.2f)"
                         % (seq, need, tasks, b, failed, tf, ta / tf))
    text = "\n".join(lines)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
