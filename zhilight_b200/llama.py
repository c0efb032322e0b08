"""Decode driver front end (zl_llama_* C-ABI).  Host buffers in, host buffers out.

Mirrors the slice of zhilight.LLaMA / DynamicBatchGenerator a decode step touches
(reference zhilight/llama.py:114-244, zhilight/dynamic_batch.py:382-639): config -> load_state_dict ->
step(tokens, positions) -> next tokens.  Scheduling (who is in the batch, at which position) stays with the
caller, exactly as the reference keeps it in src/generator.
"""
import ctypes

import numpy as np

from . import _lib
from . import beam_search as _beam
from .prefix_cache import PrefixCache

MODEL_PRESETS = {
    # SURVEY.md section 8: shapes of the BASELINE.json configs
    "llama-3.1-8b": dict(num_layers=32, dim_model=4096, num_heads=32, num_kv_heads=8, dim_head=128, dim_ff=14336,
                         vocab_size=128256, eps=1e-5, rope_theta=500000.0,
                         rope_llama3=dict(factor=8.0, low=1.0, high=4.0, orig=8192.0)),
    "llama-3.2-1b": dict(num_layers=16, dim_model=2048, num_heads=32, num_kv_heads=8, dim_head=64, dim_ff=8192,
                         vocab_size=128256, eps=1e-5, rope_theta=500000.0,
                         rope_llama3=dict(factor=32.0, low=1.0, high=4.0, orig=8192.0)),
    # north_star TP=8 target and BASELINE config 4 (Qwen2-72B GPTQ: FF padded to 29696 in the GPTQ build,
    # zhilight/config/qwen2_adapter.py:27-28; q/k/v bias, attention.cpp:105-109)
    "llama-3.1-70b": dict(num_layers=80, dim_model=8192, num_heads=64, num_kv_heads=8, dim_head=128, dim_ff=28672,
                          vocab_size=128256, eps=1e-5, rope_theta=500000.0,
                          rope_llama3=dict(factor=8.0, low=1.0, high=4.0, orig=8192.0)),
    "qwen2-72b": dict(num_layers=80, dim_model=8192, num_heads=64, num_kv_heads=8, dim_head=128, dim_ff=29696,
                      vocab_size=152064, eps=1e-6, rope_theta=1000000.0, rope_llama3=None, qkv_bias=True),
    "tiny": dict(num_layers=2, dim_model=256, num_heads=4, num_kv_heads=2, dim_head=64, dim_ff=512,
                 vocab_size=512, eps=1e-5, rope_theta=10000.0, rope_llama3=None),
}

MAX_LOGIT_BIAS = 1024   # ZL_MAX_LOGIT_BIAS


def logit_bias_arrays(logit_bias, vocab_size):
    """{token: bias} (keys may be ints or decimal strings, as in the OpenAI protocol) -> (int32 tokens, fp32 values).
    Raises ValueError for a repeated token, an id outside [0, vocab_size), a NaN or +inf bias, or more than
    MAX_LOGIT_BIAS entries; -inf bans a token."""
    items = list((logit_bias or {}).items())
    if len(items) > MAX_LOGIT_BIAS:
        raise ValueError("logit_bias has %d entries, at most %d are served" % (len(items), MAX_LOGIT_BIAS))
    toks = np.array([int(k) for k, _ in items], dtype=np.int64)
    vals = np.array([float(v) for _, v in items], dtype=np.float32)
    if np.unique(toks).size != toks.size:
        raise ValueError("logit_bias names a token twice")
    if toks.size and (toks.min() < 0 or toks.max() >= vocab_size):
        raise ValueError("logit_bias token outside [0, %d)" % vocab_size)
    if np.isnan(vals).any() or (vals == np.inf).any():
        raise ValueError("logit_bias values must be finite or -inf")
    return toks.astype(np.int32), vals


def check_ngram_penalty(ngram_penalty):
    """ngram_penalty must be finite and > 0; <= 1 turns the n-gram rule off (batch_generator.cpp:1664)."""
    if not (np.isfinite(ngram_penalty) and ngram_penalty > 0):
        raise ValueError("ngram_penalty must be finite and > 0, got %r" % (ngram_penalty,))


MAX_STOP_IDS = 8   # ZL_MAX_STOP_IDS


def stop_rule(stop_ids, max_new_tokens, vocab_size):
    """Check a stop rule for zl_llama_set_stop -> (int32 stop ids, max_new_tokens).  Raises ValueError for more than
    MAX_STOP_IDS ids, a repeated id, an id outside [0, vocab_size), or max_new_tokens < 0 (0: no budget)."""
    ids = np.asarray(list(stop_ids), dtype=np.int64).reshape(-1)
    if ids.size > MAX_STOP_IDS:
        raise ValueError("%d stop ids, at most %d are served" % (ids.size, MAX_STOP_IDS))
    if np.unique(ids).size != ids.size:
        raise ValueError("a stop id is named twice")
    if ids.size and (ids.min() < 0 or ids.max() >= vocab_size):
        raise ValueError("stop id outside [0, %d)" % vocab_size)
    if int(max_new_tokens) != max_new_tokens or max_new_tokens < 0:
        raise ValueError("max_new_tokens must be an integer >= 0 (0: no budget), got %r" % (max_new_tokens,))
    return ids.astype(np.int32), int(max_new_tokens)


KV_FULL = -5   # ZL_ERR_KV_FULL


def kv_arena_replay(kv_rows, max_batch, max_seq, ops, max_moves=1 << 16):
    """The KV arena's decisions without a device (zl_kv_arena_replay).  ops: a list of calls, each (task, rows) or a list
    of (task, rows) granted together as one entry point's call; rows >= 1 grants the task at least that many rows, 0
    releases it (alone in its call).  -> (results (n,) 0 or KV_FULL, extents (n, max_batch, 2) {first row, capacity}
    after each call, moves (m, 6) {first op of the call, launch, src, dst, rows copied, rows zero-filled}), one entry of
    results and extents per (task, rows) pair in call order."""
    lib = _lib.load()
    flat = []
    for c, call in enumerate(ops):
        pairs = [call] if np.ndim(call) == 1 else list(call)
        flat += [(c, int(t), int(r)) for t, r in pairs]
    o = np.ascontiguousarray(np.asarray(flat, dtype=np.int32).reshape(-1, 3))
    n = o.shape[0]
    res = np.empty(n, np.int32)
    ext = np.empty((n, max_batch, 2), np.int32)
    mv = np.empty((max_moves, 6), np.int32)
    nm = ctypes.c_int()
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    _lib.check(lib.zl_kv_arena_replay(int(kv_rows), int(max_batch), int(max_seq), p(o), n, p(res), p(ext), p(mv),
                                      int(max_moves), ctypes.byref(nm)))
    return res, ext, mv[:nm.value].copy()


QUANT_NONE, QUANT_AUTO_INT8, QUANT_GPTQ, QUANT_AWQ, QUANT_FP8, QUANT_FP8_BLOCK = 0, 2, 5, 6, 7, 10   # model_config.hpp:132-144


def pack_joined_segments(segments, max_batch, max_seq, vocab_size):
    """Validate the segments of a joined step, [(task, tokens, pos0, emit), ...], and pack them for zl_llama_step_joined:
    -> (tokens (sum n) int32, seg (nseg, 4) int32 {task, pos0, n, emit}).  Raises ValueError for a malformed list."""
    segments = list(segments)
    if not segments or len(segments) > max_batch:
        raise ValueError("a joined step takes 1 .. max_batch (%d) segments, not %d" % (max_batch, len(segments)))
    seg = np.zeros((len(segments), 4), dtype=np.int32)
    toks, seen = [], set()
    for i, s in enumerate(segments):
        if len(s) != 4:
            raise ValueError("segment %d: expected (task, tokens, pos0, emit)" % i)
        task, tokens, pos0, emit = s
        t = np.asarray(tokens)
        if t.ndim != 1 or t.size == 0 or not np.issubdtype(t.dtype, np.integer):
            raise ValueError("segment %d: tokens must be a non-empty 1-D integer array" % i)
        task, pos0 = int(task), int(pos0)
        if not 0 <= task < max_batch or task in seen:
            raise ValueError("segment %d: task %d out of range or repeated" % (i, task))
        if pos0 < 0 or pos0 + t.size > max_seq:
            raise ValueError("segment %d: positions %d .. %d outside the KV buffers (max_seq %d)"
                             % (i, pos0, pos0 + t.size - 1, max_seq))
        if t.min() < 0 or t.max() >= vocab_size:
            raise ValueError("segment %d: token id out of range" % i)
        seen.add(task)
        seg[i] = (task, pos0, t.size, 1 if emit else 0)
        toks.append(t.astype(np.int32))
    return np.ascontiguousarray(np.concatenate(toks)), seg


class LlamaDecoder:
    def __init__(self, num_layers, dim_model, num_heads, num_kv_heads, dim_head, dim_ff, vocab_size, eps=1e-5,
                 rope_theta=10000.0, rope_llama3=None, quant_type=QUANT_NONE, group_size=128, sym=False,
                 dtype="f16", max_batch=1, max_seq=512, use_pdl=True, use_graph=True, tp_rank=0, tp_size=1, fuse=2, tp_int8=False,
                 prefill_chunk=0, qkv_bias=False, kv_cache_dtype=None, kv_rows=None):
        """kv_cache_dtype: None keeps K/V in the activation dtype; "int8" stores them as per-(token, kv head) int8 codes
        with fp32 scales (the reference's KV_CACHE_DTYPE=int8; fp16 models with dim_head 64 or 128).
        kv_rows: None (or 0) gives every task slot max_seq KV rows for good; 1 .. max_batch * max_seq allocates that many
        rows per layer (rounded up to 64) shared by all slots, granted to each task as its writes reach them.  A call the
        arena cannot serve raises ZLError with code KV_FULL and changes nothing: release a task (kv_release) and retry."""
        if kv_cache_dtype not in (None, "int8"):
            raise ValueError("kv_cache_dtype must be None or 'int8', not %r" % (kv_cache_dtype,))
        self.lib = _lib.load()
        l3 = rope_llama3 or {}
        self.cfg = _lib.LlamaConfig(
            num_layers, dim_model, num_heads, num_kv_heads, dim_head, dim_ff, vocab_size, eps, rope_theta,
            float(l3.get("factor", 0.0)), float(l3.get("low", 1.0)), float(l3.get("high", 4.0)),
            float(l3.get("orig", 8192.0)), quant_type, group_size, int(sym), {"f16": 0, "bf16": 1}[dtype],
            max_batch, max_seq, tp_rank, tp_size, int(use_pdl), int(use_graph), int(tp_int8), int(fuse), int(prefill_chunk), int(qkv_bias),
            int(kv_cache_dtype == "int8"), int(kv_rows or 0))
        self.vocab_size = vocab_size
        self.vocab_shard = vocab_size // tp_size      # lm_head is vocab-parallel: logits come back per rank shard
        self.max_batch = max_batch
        self.kv_cache_dtype = kv_cache_dtype
        self.kv_row = (num_kv_heads // tp_size, dim_head)     # this rank's (H_kv, d) of one cached token
        self.dtype = dtype
        h = ctypes.c_void_p()
        _lib.check(self.lib.zl_llama_create(ctypes.byref(self.cfg), ctypes.byref(h)))
        self.h = h

    def set_comm(self, comm):
        """comm: zhilight_b200.dist.TPComm (kept alive by this object)."""
        self._comm = comm
        _lib.check(self.lib.zl_llama_set_comm(self.h, comm.handle))

    def enable_tp_picks(self, group=None):
        """Serve sampling, logits processors, beam_search, set_stop and generate under tensor parallelism: every rank
        gathers the lm_head shards of a sampled or beam step over NVLink and picks from the whole rows
        (zl_llama_set_vocab_gather).  Collective: every rank calls it, and from then on every rank must make the same
        set_sampling, set_stop, beam_step and generate calls, as it makes the same decode calls.  A no-op at tp_size 1."""
        if self.cfg.tp_size == 1 or getattr(self, "_vgather", None) is not None:
            return
        from .dist import VocabGather
        g = VocabGather(self.max_batch, self.vocab_size, self.cfg.tp_rank, self.cfg.tp_size, group)
        _lib.check(self.lib.zl_llama_set_vocab_gather(self.h, g.handle))
        self._vgather = g   # released after the model (close)

    def close(self):
        if getattr(self, "h", None):
            self.lib.zl_llama_destroy(self.h)
            self.h = None
        if getattr(self, "_vgather", None) is not None:
            self._vgather.close()
            self._vgather = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_state_dict(self, state_dict):
        """state_dict: name -> numpy array (2-D or 1-D), HF/ZhiLight checkpoint layout."""
        for name, arr in state_dict.items():
            a = np.ascontiguousarray(arr)
            rows, cols = (1, a.shape[0]) if a.ndim == 1 else a.shape
            _lib.check(self.lib.zl_llama_load_tensor(self.h, name.encode(), a.ctypes.data_as(ctypes.c_void_p),
                                                     rows, cols, a.itemsize))
        _lib.check(self.lib.zl_llama_finalize(self.h))

    def init_synthetic(self, seed=0):
        _lib.check(self.lib.zl_llama_init_synthetic(self.h, seed))

    def decode(self, tokens, positions, want_logits=False):
        """One step: tokens/positions int32 host arrays (B).  Returns next tokens (B) [, logits (B, V/tp) fp32: this
        rank's vocabulary shard]."""
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        p = np.ascontiguousarray(positions, dtype=np.int32)
        b = t.size
        nxt = np.empty(b, dtype=np.int32)
        logits = np.empty((b, self.vocab_shard), dtype=np.float32) if want_logits else None
        _lib.check(self.lib.zl_llama_decode(
            self.h, t.ctypes.data_as(ctypes.c_void_p), p.ctypes.data_as(ctypes.c_void_p), b,
            nxt.ctypes.data_as(ctypes.c_void_p),
            logits.ctypes.data_as(ctypes.c_void_p) if want_logits else None))
        return (nxt, logits) if want_logits else nxt

    def prefill(self, task, tokens, pos0=0, want_logits=False):
        """Chunked prefill of one task's prompt; returns the next token (greedy, or sampled per set_sampling)
        [, logits of the last position]."""
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        nxt = np.empty(1, dtype=np.int32)
        logits = np.empty((1, self.vocab_shard), dtype=np.float32) if want_logits else None
        _lib.check(self.lib.zl_llama_prefill(
            self.h, int(task), t.ctypes.data_as(ctypes.c_void_p), t.size, int(pos0),
            nxt.ctypes.data_as(ctypes.c_void_p), logits.ctypes.data_as(ctypes.c_void_p) if want_logits else None))
        return (int(nxt[0]), logits) if want_logits else int(nxt[0])

    def step_joined(self, segments, want_logits=False):
        """One joined step (zl_llama_step_joined): segments = [(task, tokens, pos0, emit), ...] of distinct tasks -- prompt
        chunks and decode rows (one token) alike -- run through one forward; rows sum(len(tokens)) <= max(max_batch,
        prefill_chunk).  Returns the next tokens (nseg,) int32, -1 where emit is false [, logits (n_emit, V/tp) fp32 of
        the emitting segments' last rows, in segment order]."""
        cfg = self.cfg
        tokens, seg = pack_joined_segments(segments, cfg.max_batch, cfg.max_seq, cfg.vocab_size)
        n_emit = int(seg[:, 3].sum())
        nxt = np.empty(seg.shape[0], dtype=np.int32)
        logits = np.empty((n_emit, self.vocab_shard), dtype=np.float32) if want_logits else None
        _lib.check(self.lib.zl_llama_step_joined(
            self.h, tokens.ctypes.data_as(ctypes.c_void_p), seg.ctypes.data_as(ctypes.c_void_p), seg.shape[0],
            nxt.ctypes.data_as(ctypes.c_void_p),
            logits.ctypes.data_as(ctypes.c_void_p) if want_logits and n_emit else None))
        return (nxt, logits) if want_logits else nxt

    def enable_prefix_cache(self, num_blocks, block_tokens=128):
        """Prompt prefix caching: a device pool of num_blocks blocks of block_tokens (16 .. 256) KV rows of every layer
        (zl_llama_kv_pool_create) and the host policy that fills it (prefix_cache.PrefixCache).  Call after the weights
        are loaded; once per model."""
        _lib.check(self.lib.zl_llama_kv_pool_create(self.h, int(num_blocks), int(block_tokens)))
        self.prefix_cache = PrefixCache(num_blocks, block_tokens)

    def _kv_blocks(self, fn, task, task_blocks, pool_blocks):
        tb = np.ascontiguousarray(task_blocks, dtype=np.int32).reshape(-1)
        pb = np.ascontiguousarray(pool_blocks, dtype=np.int32).reshape(-1)
        if tb.size != pb.size:
            raise ValueError("task_blocks and pool_blocks differ in length (%d, %d)" % (tb.size, pb.size))
        if tb.size:
            _lib.check(fn(self.h, int(task), tb.ctypes.data_as(ctypes.c_void_p), pb.ctypes.data_as(ctypes.c_void_p),
                          tb.size))

    def kv_save_blocks(self, task, task_blocks, pool_blocks):
        """Copy the task's blocks task_blocks[i] (rows [j bt, (j + 1) bt)) into pool blocks pool_blocks[i], every layer;
        stream-ordered after the steps already issued (zl_llama_kv_blocks_save)."""
        self._kv_blocks(self.lib.zl_llama_kv_blocks_save, task, task_blocks, pool_blocks)

    def kv_load_blocks(self, task, task_blocks, pool_blocks):
        """Copy pool blocks pool_blocks[i] into the task's blocks task_blocks[i] (zl_llama_kv_blocks_load).  Writes KV rows
        only: continue with prefill(task, rest, pos0=loaded length) or a step_joined segment at that position."""
        self._kv_blocks(self.lib.zl_llama_kv_blocks_load, task, task_blocks, pool_blocks)

    def prefill_cached(self, task, tokens, want_logits=False):
        """prefill() through the prefix cache: load the longest cached prefix of `tokens` into the task, prefill the
        rest at pos0 = its length, then cache the prompt's new blocks.  Returns (next token, cached length
        [, logits]).  A cached row holds the bits of the prefill that wrote it, so the logits can differ in their last
        bits from a cold prefill that split the prompt into different chunks."""
        pc = getattr(self, "prefix_cache", None)
        if pc is None:
            raise RuntimeError("prefill_cached needs enable_prefix_cache() first")
        t = np.ascontiguousarray(tokens, dtype=np.int32).reshape(-1)
        hit = pc.match(t)
        self.kv_load_blocks(task, range(len(hit)), hit)
        m = len(hit) * pc.block_tokens
        out = self.prefill(task, t[m:], pos0=m, want_logits=want_logits)
        save = pc.insert(t)
        self.kv_save_blocks(task, [j for j, _ in save], [b for _, b in save])
        return (out[0], m, out[1]) if want_logits else (out, m)

    def bench_kv_blocks(self, task, task_blocks, pool_blocks, load=True, per_range_memcpy=False, iters=20):
        """-> (ms per pass, bytes one pass reads plus writes) of `iters` timed block copies (zl_llama_kv_blocks_bench)."""
        tb = np.ascontiguousarray(task_blocks, dtype=np.int32)
        pb = np.ascontiguousarray(pool_blocks, dtype=np.int32)
        ms, by = ctypes.c_float(), ctypes.c_double()
        _lib.check(self.lib.zl_llama_kv_blocks_bench(
            self.h, int(task), tb.ctypes.data_as(ctypes.c_void_p), pb.ctypes.data_as(ctypes.c_void_p), tb.size,
            int(bool(load)), int(bool(per_range_memcpy)), int(iters), ctypes.byref(ms), ctypes.byref(by)))
        return ms.value / iters, by.value

    def beam_step(self, tokens, positions, groups, cum, k, want_logits=False):
        """One beam step (zl_llama_beam_step): the decode step over tasks 0 .. B-1 with zl_beam_topk as its pick.
        groups (G, 2) {row0, width} tile the rows; cum (B) the rows' cumulative log-probabilities (-inf: dead row).
        Returns (parent, token, score), each (G, k) [, logits (B, V)]."""
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        p = np.ascontiguousarray(positions, dtype=np.int32)
        g = np.ascontiguousarray(groups, dtype=np.int32).reshape(-1, 2)
        c = np.ascontiguousarray(cum, dtype=np.float32)
        if c.size != t.size or p.size != t.size:
            raise ValueError("tokens, positions and cum differ in length (%d, %d, %d)" % (t.size, p.size, c.size))
        n, k = g.shape[0], int(k)
        parent = np.empty((n, max(k, 0)), np.int32)
        token = np.empty_like(parent)
        score = np.empty((n, max(k, 0)), np.float32)
        logits = np.empty((t.size, self.vocab_shard), dtype=np.float32) if want_logits else None
        ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        _lib.check(self.lib.zl_llama_beam_step(self.h, ptr(t), ptr(p), t.size, ptr(g), n, ptr(c), k, ptr(parent),
                                               ptr(token), ptr(score), ptr(logits) if want_logits else None))
        return (parent, token, score, logits) if want_logits else (parent, token, score)

    def kv_copy_rows(self, ranges):
        """Copy KV rows between tasks, every layer (zl_llama_kv_copy_rows): ranges (n, 4) {src task, dst task, row0, row1};
        stream-ordered after the steps already issued."""
        r = np.ascontiguousarray(ranges, dtype=np.int32).reshape(-1, 4)
        if r.shape[0]:
            _lib.check(self.lib.zl_llama_kv_copy_rows(self.h, r.ctypes.data_as(ctypes.c_void_p), r.shape[0]))

    def beam_search(self, prompts, beam_width, max_new_tokens, eos_id, num_results=1, trace=None):
        """Beam search (beam_search.beam_search) over prompts, prompt g in tasks [g W, (g + 1) W): needs
        max_batch >= len(prompts) * beam_width and, for prompts longer than one token, prefill_chunk > 0.  Returns per
        prompt up to num_results (tokens, score, cum_logprob) best first; score = cum_logprob / len(tokens + EOS)."""
        need = len(prompts) * int(beam_width)
        if need > self.max_batch:
            raise ValueError("beam search over %d prompts of width %d needs max_batch >= %d (have %d)"
                             % (len(prompts), beam_width, need, self.max_batch))
        if self.cfg.prefill_chunk <= 0 and any(len(p) > 1 for p in prompts):
            raise ValueError("beam search over prompts longer than one token needs prefill_chunk > 0")
        return _beam.beam_search(
            lambda t, p, g, c, k: self.beam_step(t, p, g, c, k), self.kv_copy_rows,
            lambda s, toks: self.prefill(s, toks), prompts, beam_width, max_new_tokens, eos_id, num_results, trace)

    def set_sampling(self, task, temperature=0.0, top_p=1.0, top_k=0, repetition_penalty=1.0, presence_penalty=0.0,
                     seed=0, ngram_penalty=1.0, logit_bias=None):
        """Per-task sampling and logits processors for the following steps (zl_llama_set_sampling, then
        zl_llama_set_logits_processors); clears the task's penalty history and generated-token sequence.  Both are set on
        every call, so a reused task slot never keeps an earlier request's bias.  logit_bias: {token: bias} or None.
        As GeneratorArg (zhilight/dynamic_batch.py:110-111), ngram_penalty is 1 when presence_penalty != 0.
        The defaults are plain greedy.  A task's constraint (set_constraint) is left alone."""
        check_ngram_penalty(ngram_penalty)
        ngram = 1.0 if presence_penalty else float(ngram_penalty)
        toks, vals = logit_bias_arrays(logit_bias, self.cfg.vocab_size)
        if self.cfg.tp_size > 1 and getattr(self, "_vgather", None) is None and (ngram > 1 or toks.size):
            # refused here so that neither the sampling nor the processors change (enable_tp_picks serves them)
            raise _lib.ZLError(-2, "logits processors under tensor parallelism need enable_tp_picks()")
        p = _lib.sample_params(temperature, top_p, top_k, repetition_penalty, presence_penalty, seed)
        _lib.check(self.lib.zl_llama_set_sampling(self.h, int(task), ctypes.byref(p)))
        _lib.check(self.lib.zl_llama_set_logits_processors(self.h, int(task), ngram, toks.ctypes.data_as(ctypes.c_void_p),
                                                           vals.ctypes.data_as(ctypes.c_void_p), toks.size))

    def enable_constraints(self, max_states, max_edges=0):
        """Device storage for one token automaton per task of up to max_states states and max_edges edges
        (zl_llama_enable_constraints); once per decoder."""
        _lib.check(self.lib.zl_llama_enable_constraints(self.h, int(max_states), int(max_edges)))

    def set_constraint(self, task, automaton):
        """Constrain the picks of `task` by a constraints.TokenAutomaton from its start state, or clear its constraint
        with None (zl_llama_set_constraint).  Every pick the task records is masked by its state's allowed set and moves
        the state on the device, in decode, step_device, prefill, step_joined and generate alike."""
        if automaton is None:
            _lib.check(self.lib.zl_llama_set_constraint(self.h, int(task), 0, None, None, 0, None, None, None, 0))
            return
        a = automaton
        if a.vocab_size != self.cfg.vocab_size:
            raise ValueError("automaton over %d tokens for a %d-token model" % (a.vocab_size, self.cfg.vocab_size))
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
        _lib.check(self.lib.zl_llama_set_constraint(self.h, int(task), a.n_states, p(a.masks), p(a.row_ptr), a.n_edges,
                                                    p(a.edge_tok), p(a.edge_next), p(a.default_next), a.start))

    def constraint_state(self, b):
        """The automaton state of tasks 0 .. b-1 (-1: unconstrained), once every enqueued step has run."""
        out = np.empty(int(b), np.int32)
        _lib.check(self.lib.zl_llama_get_constraint_state(self.h, out.ctypes.data_as(ctypes.c_void_p), int(b)))
        return out

    def kv_release(self, task):
        """Return the task's KV rows to the arena; its next write is granted fresh, zero-filled rows
        (zl_llama_kv_release).  A no-op without kv_rows."""
        _lib.check(self.lib.zl_llama_kv_release(self.h, int(task)))

    def kv_capacity(self, task):
        """KV rows the task holds now (max_seq without kv_rows)."""
        r = ctypes.c_int()
        _lib.check(self.lib.zl_llama_kv_capacity(self.h, int(task), ctypes.byref(r)))
        return r.value

    def kv_free_rows(self):
        """KV rows of the arena no task holds (0 without kv_rows)."""
        r = ctypes.c_int()
        _lib.check(self.lib.zl_llama_kv_free_rows(self.h, ctypes.byref(r)))
        return r.value

    def read_kv(self, layer, task, row0, n):
        """Rows row0 .. row0 + n of a task's layer-`layer` KV cache (zl_llama_read_kv), each (n, H_kv, d).
        Plain cache: (k, v) as float16 (bf16 models: uint16 bit patterns).  int8 cache: (k, v, scale_k, scale_v) with
        uint8 codes and (n, H_kv) float32 scales; a value is (code - 128) * scale."""
        hkv, d = self.kv_row
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        if self.kv_cache_dtype == "int8":
            k, v = np.empty((n, hkv, d), np.uint8), np.empty((n, hkv, d), np.uint8)
            sk, sv = np.empty((n, hkv), np.float32), np.empty((n, hkv), np.float32)
            _lib.check(self.lib.zl_llama_read_kv(self.h, layer, task, row0, n, p(k), p(v), p(sk), p(sv)))
            return k, v, sk, sv
        dt = np.float16 if self.dtype == "f16" else np.uint16
        k, v = np.empty((n, hkv, d), dt), np.empty((n, hkv, d), dt)
        _lib.check(self.lib.zl_llama_read_kv(self.h, layer, task, row0, n, p(k), p(v), None, None))
        return k, v

    def set_state(self, tokens, positions):
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        p = np.ascontiguousarray(positions, dtype=np.int32)
        _lib.check(self.lib.zl_llama_set_state(self.h, t.ctypes.data_as(ctypes.c_void_p),
                                               p.ctypes.data_as(ctypes.c_void_p), t.size))

    def get_state(self, b):
        t = np.empty(b, dtype=np.int32)
        p = np.empty(b, dtype=np.int32)
        _lib.check(self.lib.zl_llama_get_state(self.h, t.ctypes.data_as(ctypes.c_void_p),
                                               p.ctypes.data_as(ctypes.c_void_p), b))
        return t, p

    def get_logits(self, b):
        """fp32 logits (b, V/tp) of the last step, this rank's vocabulary shard."""
        out = np.empty((b, self.vocab_shard), dtype=np.float32)
        _lib.check(self.lib.zl_llama_get_logits(self.h, out.ctypes.data_as(ctypes.c_void_p), b))
        return out

    def step_device(self, b):
        _lib.check(self.lib.zl_llama_step_device(self.h, b))

    def set_stop(self, task, stop_ids=(), max_new_tokens=0):
        """The stop rule of `task` for generate(): it finishes when it emits one of stop_ids (at most MAX_STOP_IDS
        distinct ids, e.g. the EOS ids) or after max_new_tokens emitted tokens (0: no budget), and always when its KV
        buffer is full.  Re-arms a finished task and restarts its count (zl_llama_set_stop)."""
        ids, budget = stop_rule(stop_ids, max_new_tokens, self.cfg.vocab_size)
        _lib.check(self.lib.zl_llama_set_stop(self.h, int(task), ids.ctypes.data_as(ctypes.c_void_p), ids.size, budget))

    def generate(self, b, max_steps):
        """Up to max_steps device-resident decode steps of tasks 0 .. b-1 from their (token, position) state
        (set_state, or earlier steps), ending early once every task has finished (zl_llama_generate).  Returns
        (list of b int32 arrays: the tokens each task emitted, stop ids included; finish reasons (b,) int32: 0 running,
        1 stop id, 2 max_new_tokens, 3 KV buffer full; steps run).  Call again to continue: the state stays on the
        device."""
        b, max_steps = int(b), int(max_steps)
        toks = np.empty((max(max_steps, 0), max(b, 0)), np.int32)
        n_out = np.empty(max(b, 0), np.int32)
        fin = np.empty(max(b, 0), np.int32)
        steps = ctypes.c_int()
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        _lib.check(self.lib.zl_llama_generate(self.h, b, max_steps, p(toks), p(n_out), p(fin), ctypes.byref(steps)))
        out = [toks[:steps.value, i][toks[:steps.value, i] >= 0].copy() for i in range(b)]
        return out, fin, steps.value

    def sync(self):
        _lib.check(self.lib.zl_llama_sync(self.h))

    def stream(self):
        return self.lib.zl_llama_stream(self.h)

    def bench_gemms(self, b=1, iters=5):
        """-> (ms for `iters` passes, GEMM launches per pass, algorithmic bytes per pass)."""
        ms = ctypes.c_float()
        n = ctypes.c_int()
        by = ctypes.c_double()
        _lib.check(self.lib.zl_llama_bench_gemms(self.h, b, iters, ctypes.byref(ms), ctypes.byref(n), ctypes.byref(by)))
        return ms.value, n.value, by.value

    def stats(self, b=1):
        wb = ctypes.c_double()
        kn = ctypes.c_int()
        _lib.check(self.lib.zl_llama_stats(self.h, b, ctypes.byref(wb), ctypes.byref(kn)))
        return wb.value, kn.value
