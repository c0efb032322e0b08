"""Decode driver front end (zl_llama_* C-ABI).  Host buffers in, host buffers out.

Mirrors the slice of zhilight.LLaMA / DynamicBatchGenerator a decode step touches
(reference zhilight/llama.py:114-244, zhilight/dynamic_batch.py:382-639): config -> load_state_dict ->
step(tokens, positions) -> next tokens.  Scheduling (who is in the batch, at which position) stays with the
caller, exactly as the reference keeps it in src/generator.
"""
import ctypes

import numpy as np

from . import _lib

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
                 prefill_chunk=0, qkv_bias=False, kv_cache_dtype=None):
        """kv_cache_dtype: None keeps K/V in the activation dtype; "int8" stores them as per-(token, kv head) int8 codes
        with fp32 scales (the reference's KV_CACHE_DTYPE=int8; fp16 models with dim_head 64 or 128)."""
        if kv_cache_dtype not in (None, "int8"):
            raise ValueError("kv_cache_dtype must be None or 'int8', not %r" % (kv_cache_dtype,))
        self.lib = _lib.load()
        l3 = rope_llama3 or {}
        self.cfg = _lib.LlamaConfig(
            num_layers, dim_model, num_heads, num_kv_heads, dim_head, dim_ff, vocab_size, eps, rope_theta,
            float(l3.get("factor", 0.0)), float(l3.get("low", 1.0)), float(l3.get("high", 4.0)),
            float(l3.get("orig", 8192.0)), quant_type, group_size, int(sym), {"f16": 0, "bf16": 1}[dtype],
            max_batch, max_seq, tp_rank, tp_size, int(use_pdl), int(use_graph), int(tp_int8), int(fuse), int(prefill_chunk), int(qkv_bias),
            int(kv_cache_dtype == "int8"))
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

    def close(self):
        if getattr(self, "h", None):
            self.lib.zl_llama_destroy(self.h)
            self.h = None

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

    def set_sampling(self, task, temperature=0.0, top_p=1.0, top_k=0, repetition_penalty=1.0, presence_penalty=0.0,
                     seed=0):
        """Per-task sampling for the following steps (zl_llama_set_sampling); clears the task's penalty history.
        The defaults are plain greedy."""
        p = _lib.sample_params(temperature, top_p, top_k, repetition_penalty, presence_penalty, seed)
        _lib.check(self.lib.zl_llama_set_sampling(self.h, int(task), ctypes.byref(p)))

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
