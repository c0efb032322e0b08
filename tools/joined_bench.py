"""Joined steps: the causal variable-length attention kernel against the masked decode kernel, and the decode driver's
joined steps against prefill-then-decode when a long prompt arrives beside running tasks.

  1. kernel: zl_varlen_attention vs zl_decode_attention(len_q = chunk, int8 causal mask), Llama-3.1-8B heads (32 / 8,
     d = 128, fp16): one chunk of 16 / 128 / 512 rows at pos0 0 / 1024 / 4096, and decode-only segment sets (B = 1 / 8 / 32
     at ctx 2048).  Median us over alternating runs, algorithmic K/V GB/s (each task's K and V rows read once), rel L2
     between the two outputs.
  2. driver: Llama-3.1-8B GPTQ-int4 (synthetic weights), prefill_chunk 512.  B tasks decode at ctx 1024 when a 2048-token
     prompt arrives: (a) 4 x zl_llama_prefill chunks of 512, then decode steps; (b) joined steps of B decode rows + (512 -
     B) prompt rows until the prompt is consumed (the reference's chunk_size_adj).  Both windows give every running task
     the same number of tokens; reported: the new prompt's TTFT, the running tasks' longest gap between two tokens, and
     tokens/s over the window (host wall clock around the synchronous calls; medians of alternating runs).

    python tools/joined_bench.py [--out FILE] [--reps 5]
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

HQ, HKV, D = 32, 8, 128
CHUNKS = (16, 128, 512)
POS0S = (0, 1024, 4096)
DECODE_BS = (1, 8, 32)
DECODE_CTX = 2048


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


class KernelCase:
    """Pre-allocated inputs of one shape for both kernels (no allocation or sync inside the timed calls)."""

    def __init__(self, torch, lens, chunk):
        from zhilight_b200 import _lib, ops
        dev = torch.device("cuda:0")
        g = torch.Generator(device=dev).manual_seed(0)
        self.torch, self.lib, self.chunk = torch, _lib.load(), chunk
        self.B = len(lens)
        self.lens = lens
        rows = chunk if chunk else self.B
        self.k = [torch.randn(n, HKV, D, device=dev, generator=g).half() for n in lens]
        self.v = [torch.randn(n, HKV, D, device=dev, generator=g).half() for n in lens]
        self.ka, self.va = ops._ptr_table(self.k, dev), ops._ptr_table(self.v, dev)
        self.q = torch.randn(rows, HQ, D, device=dev, generator=g).half()
        self.out_va, self.out_da = torch.empty_like(self.q), torch.empty_like(self.q)
        self.max_keys = max(lens)
        if chunk:   # one segment: the chunk's rows are the last `chunk` positions of task 0
            pos0 = lens[0] - chunk
            seg = [(0, 0, pos0, chunk)]
            mask = (np.arange(lens[0])[None, :] <= pos0 + np.arange(chunk)[:, None]).astype(np.int8)
            self.mask = torch.from_numpy(mask.reshape(-1)).to(dev)
            self.len_q = chunk
        else:       # decode rows: task b at position lens[b] - 1
            seg = [(b, b, n - 1, 1) for b, n in enumerate(lens)]
            self.mask = None
            self.len_q = 1
        self.seg = torch.tensor(seg, dtype=torch.int32, device=dev)
        self.buf_lens = torch.tensor(lens, dtype=torch.int32, device=dev)
        self.va_ws_bytes = self.lib.zl_varlen_attention_workspace_bytes(rows, len(seg), HQ, D, self.max_keys)
        self.da_ws_bytes = self.lib.zl_decode_attention_workspace_bytes(self.B, self.len_q, HQ, D, self.max_keys)
        self.va_ws = torch.empty(max(1, self.va_ws_bytes), dtype=torch.uint8, device=dev)
        self.da_ws = torch.empty(max(1, self.da_ws_bytes), dtype=torch.uint8, device=dev)
        self.rows = rows
        self.kv_bytes = sum(2.0 * n * HKV * D * 2 for n in lens)

    def varlen(self):
        from zhilight_b200 import _lib
        _lib.check(self.lib.zl_varlen_attention(_ptr(self.q), _ptr(self.seg), self.seg.shape[0], self.rows, _ptr(self.ka),
                                                _ptr(self.va), 1.0 / np.sqrt(D), self.max_keys, _ptr(self.out_va), HQ, HKV,
                                                D, _ptr(self.va_ws), self.va_ws_bytes, 0, 0, self._stream()))

    def decode(self):
        from zhilight_b200 import _lib
        m = _ptr(self.mask) if self.mask is not None else None
        _lib.check(self.lib.zl_decode_attention(_ptr(self.q), _ptr(self.buf_lens), _ptr(self.ka), _ptr(self.va), m,
                                                1.0 / np.sqrt(D), self.max_keys, _ptr(self.out_da), self.B, self.len_q,
                                                HQ, HKV, D, 1, _ptr(self.da_ws), self.da_ws_bytes, 0, 0, self._stream()))

    def _stream(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream().cuda_stream)


def time_us(torch, fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / iters


def kernel_part(torch, reps, log):
    from tests.helpers import rel_l2
    log("## one attention launch, Llama-3.1-8B heads (32 q / 8 kv, d = 128, fp16): us per call, median (min-max) of %d "
        "alternating runs; GB/s = algorithmic K/V bytes (each task's rows read once) / time" % reps)
    cases = [("chunk %3d pos0 %4d" % (c, p), [p + c], c) for c in CHUNKS for p in POS0S]
    cases += [("decode B=%-2d ctx %d" % (b, DECODE_CTX), [DECODE_CTX] * b, 0) for b in DECODE_BS]
    for name, lens, chunk in cases:
        kc = KernelCase(torch, lens, chunk)
        iters = 20 if kc.rows * max(lens) > 1 << 20 else 200
        res = {"varlen": [], "decode": []}
        for _ in range(reps):
            res["varlen"].append(time_us(torch, kc.varlen, iters))
            res["decode"].append(time_us(torch, kc.decode, iters))
        torch.cuda.synchronize()
        err = rel_l2(kc.out_va.float().cpu().numpy(), kc.out_da.float().cpu().numpy())
        mv, md = statistics.median(res["varlen"]), statistics.median(res["decode"])
        log("%s  varlen %9.2f us (%.2f-%.2f) %6.0f GB/s  masked decode kernel %9.2f us (%.2f-%.2f) %6.0f GB/s  "
            "decode/varlen %6.2fx  rel L2 %.1e"
            % (name, mv, min(res["varlen"]), max(res["varlen"]), kc.kv_bytes / mv / 1e3, md, min(res["decode"]),
               max(res["decode"]), kc.kv_bytes / md / 1e3, md / mv, err))
        del kc
        torch.cuda.empty_cache()


def driver_part(torch, reps, log):
    from zhilight_b200.llama import MODEL_PRESETS, LlamaDecoder
    cfg = MODEL_PRESETS["llama-3.1-8b"]
    V = cfg["vocab_size"]
    chunk, prompt_len, ctx = 512, 2048, 1024
    max_b = max(DECODE_BS)
    dec = LlamaDecoder(quant_type=5, group_size=128, sym=True, max_batch=max_b + 1, max_seq=ctx + prompt_len + 64,
                       prefill_chunk=chunk, **cfg)
    dec.init_synthetic(0)
    rng = np.random.default_rng(0)
    prompt = rng.integers(0, V, prompt_len).astype(np.int32)
    log("## driver: Llama-3.1-8B GPTQ-int4 (synthetic, sym), prefill_chunk %d; B tasks decoding at ctx %d when a %d-token "
        "prompt arrives (task B).  (a) 4 x zl_llama_prefill(512) then decode steps; (b) joined steps of B decode rows + "
        "(512 - B) prompt rows.  Both windows give every running task J tokens (J = joined steps needed for the prompt). "
        "ms, median (min-max) of %d alternating runs, host wall clock around synchronous calls" % (chunk, ctx, prompt_len,
                                                                                                 reps))

    def run_a(B, J):
        pos = np.full(B, ctx, np.int32)
        tok = rng.integers(0, V, B).astype(np.int32)
        dec.decode(tok, pos)                 # the running tasks' token just before the prompt arrives
        pos += 1
        t0 = time.perf_counter()
        last_tok = t0
        gap = 0.0
        for c in range(prompt_len // chunk):
            dec.prefill(B, prompt[c * chunk:(c + 1) * chunk], pos0=c * chunk)
        ttft = time.perf_counter() - t0
        for _ in range(J):
            tok = dec.decode(tok, pos)
            pos += 1
            now = time.perf_counter()
            gap = max(gap, now - last_tok)
            last_tok = now
        return ttft, gap, (B * J + 1) / (last_tok - t0), None

    def run_b(B, J):
        pos = np.full(B, ctx, np.int32)
        tok = rng.integers(0, V, B).astype(np.int32)
        dec.decode(tok, pos)
        pos += 1
        per = chunk - B
        t0 = time.perf_counter()
        last_tok = t0
        gap, ttft, off = 0.0, None, 0
        steps = []
        for _ in range(J):
            segs = [(t, tok[t:t + 1], int(pos[t]), True) for t in range(B)]
            if off < prompt_len:
                n = min(per, prompt_len - off)
                segs.append((B, prompt[off:off + n], off, off + n == prompt_len))
                off += n
            s0 = time.perf_counter()
            nxt = dec.step_joined(segs)
            now = time.perf_counter()
            steps.append(now - s0)
            tok = nxt[:B].astype(np.int32)
            pos += 1
            gap = max(gap, now - last_tok)
            last_tok = now
            if ttft is None and off >= prompt_len:
                ttft = now - t0
        return ttft, gap, (B * J + 1) / (last_tok - t0), steps

    for B in DECODE_BS:
        J = -(-prompt_len // (chunk - B))
        res = {"a": [], "b": []}
        step_b = []
        for _ in range(reps):
            res["a"].append(run_a(B, J))
            r = run_b(B, J)
            res["b"].append(r)
            step_b.append(statistics.median(r[3]))
        row = []
        for k, label in ((0, "TTFT ms"), (1, "longest gap ms"), (2, "tok/s")):
            sc = 1e3 if k < 2 else 1.0
            a = [x[k] * sc for x in res["a"]]
            b = [x[k] * sc for x in res["b"]]
            row.append("%s (a) %.1f (%.1f-%.1f) (b) %.1f (%.1f-%.1f)" % (label, statistics.median(a), min(a), max(a),
                                                                      statistics.median(b), min(b), max(b)))
        log("B=%-2d J=%d  %s" % (B, J, "  ".join(row)))
        log("      joined step (B decode + %d prompt rows) median %.2f ms" % (chunk - B, 1e3 * statistics.median(step_b)))
    # one 512-token prefill chunk against one joined step of 8 decode + 504 prompt rows, alternating
    pf, jn = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        dec.prefill(max_b, prompt[:chunk], pos0=0)
        pf.append(time.perf_counter() - t0)
        segs = [(t, np.array([1], np.int32), ctx, True) for t in range(8)] + [(max_b, prompt[:chunk - 8], 0, False)]
        t0 = time.perf_counter()
        dec.step_joined(segs)
        jn.append(time.perf_counter() - t0)
    log("one zl_llama_prefill chunk of 512 rows %.2f ms (%.2f-%.2f)  one joined step of 8 decode + 504 prompt rows %.2f ms "
        "(%.2f-%.2f)  joined/prefill %.3f" % (1e3 * statistics.median(pf), 1e3 * min(pf), 1e3 * max(pf),
                                              1e3 * statistics.median(jn), 1e3 * min(jn), 1e3 * max(jn),
                                              statistics.median(jn) / statistics.median(pf)))
    dec.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-driver", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("joined_bench needs a CUDA device")
    from zhilight_b200 import build
    build.build()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    log("card: %s" % card())
    kernel_part(torch, args.reps, log)
    if not args.skip_driver:
        driver_part(torch, args.reps, log)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
