"""GPU parity of joined steps (zl_llama_step_joined): running tasks' decode rows and another task's prompt chunks in one
forward, against the CPU oracle model fed token by token, for every weight format the driver serves."""
import ctypes

import numpy as np
import pytest

from oracle import model as omodel
from tests import sampling_oracle as so
from tests.helpers import from_bf16_bits, rel_l2
from tests.test_llama_gpu import LAYER8B, TINY, TINY128
from tests.test_sampling_gpu import _sample

pytestmark = pytest.mark.gpu

PREFIX = (5, 9, 3)   # prompt lengths of tasks 0-2, prefilled before the joined steps


def _decoder(cfg, quant, dtype, sd, sym=False, prefill_chunk=48, **kw):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=quant, dtype=dtype, sym=sym, max_batch=4, max_seq=128, prefill_chunk=prefill_chunk,
                       **cfg, **kw)
    dec.load_state_dict(sd)
    return dec


def _scenario(cfg, quant, dtype, tol, chunks, sym=False, scale_range=None, seed=0, check_kv=False):
    """Tasks 0-2 are prefilled; joined steps then carry their decode rows plus task 3's prompt in `chunks` (emit on the
    last); decoding continues in a joined step and in plain decode steps.  Every emitted logits row matches the oracle."""
    sd = omodel.make_state_dict(cfg, quant, 128, sym, seed=seed, dtype=dtype, scale_range=scale_range)
    dec = _decoder(cfg, quant, dtype, sd, sym=sym)
    orc = omodel.OracleLlama(cfg, sd, quant, 128, sym, dtype, fuse_norm=True)
    rng = np.random.default_rng(seed)
    V = cfg["vocab_size"]
    pos = np.zeros(4, np.int32)
    fed = {t: [] for t in range(4)}       # (token, position) of every row written, for the KV comparison
    for t, n in enumerate(PREFIX):
        prompt = rng.integers(0, V, n).astype(np.int32)
        _, lg = dec.prefill(t, prompt, want_logits=True)
        for p, tok in enumerate(prompt):
            r = orc.decode(prompt[p:p + 1], [p], tasks=[t])
        assert rel_l2(lg, r) <= tol
        fed[t] += [(int(x), p) for p, x in enumerate(prompt)]
        pos[t] = n
    prompt3 = rng.integers(0, V, sum(chunks)).astype(np.int32)
    off = 0
    for i, cn in enumerate(chunks):
        last = i == len(chunks) - 1
        tok = rng.integers(0, V, 3).astype(np.int32)
        segs = [(t, tok[t:t + 1], int(pos[t]), True) for t in range(3)] + [(3, prompt3[off:off + cn], off, last)]
        nxt, logits = dec.step_joined(segs, want_logits=True)
        ref = orc.decode(tok, pos[:3], tasks=[0, 1, 2])
        for p in range(off, off + cn):
            r3 = orc.decode(prompt3[p:p + 1], [p], tasks=[3])
        assert logits.shape == (4 if last else 3, V)
        assert rel_l2(logits[:3], ref) <= tol, i      # the decode rows, as the decode tests compare a batch
        for t in range(3):
            assert nxt[t] == int(np.argmax(logits[t]))
            fed[t].append((int(tok[t]), int(pos[t])))
        if last:
            assert rel_l2(logits[3], r3[0]) <= tol
            assert nxt[3] == int(np.argmax(logits[3]))
        else:
            assert nxt[3] == -1
        fed[3] += [(int(x), off + j) for j, x in enumerate(prompt3[off:off + cn])]
        pos[:3] += 1
        off += cn
    pos[3] = off
    # a joined step of decode rows only, then plain decode steps
    tok = rng.integers(0, V, 4).astype(np.int32)
    nxt, logits = dec.step_joined([(t, tok[t:t + 1], int(pos[t]), True) for t in range(4)], want_logits=True)
    ref = orc.decode(tok, pos, tasks=[0, 1, 2, 3])
    assert rel_l2(logits, ref) <= tol
    for t in range(4):
        fed[t].append((int(tok[t]), int(pos[t])))
    pos += 1
    for _ in range(2):
        tok = rng.integers(0, V, 4).astype(np.int32)
        nxt, logits = dec.decode(tok, pos, want_logits=True)
        ref = orc.decode(tok, pos, tasks=[0, 1, 2, 3])
        assert rel_l2(logits, ref) <= tol
        for t in range(4):
            fed[t].append((int(tok[t]), int(pos[t])))
        pos += 1
    if check_kv:
        # the same rows written by zl_llama_prefill + zl_llama_decode
        ref_dec = _decoder(cfg, quant, dtype, sd, sym=sym)
        for t in range(4):
            n_pf = PREFIX[t] if t < 3 else len(prompt3)
            ref_dec.prefill(t, np.array([x for x, _ in fed[t][:n_pf]], np.int32))
        for s in range(max(len(f) for f in fed.values()) - min(PREFIX)):
            rows = [(t, fed[t][(PREFIX[t] if t < 3 else len(prompt3)) + s]) for t in range(4)
                    if (PREFIX[t] if t < 3 else len(prompt3)) + s < len(fed[t])]
            if not rows:
                break
            # decode runs tasks 0 .. B-1: give every task its row or a dummy write far past the compared range
            b = max(t for t, _ in rows) + 1
            tk = np.zeros(b, np.int32)
            ps = np.full(b, 120, np.int32)
            for t, (x, p) in rows:
                tk[t], ps[t] = x, p
            ref_dec.decode(tk, ps)
        for t in range(4):
            n = len(fed[t])
            k, v = dec.read_kv(0, t, 0, n)
            rk, rv = ref_dec.read_kv(0, t, 0, n)
            f = (lambda a: a.astype(np.float32)) if dtype == "f16" else from_bf16_bits
            assert rel_l2(f(k), f(rk)) <= tol and rel_l2(f(v), f(rv)) <= tol, t
        ref_dec.close()
    return dec


@pytest.mark.parametrize("cfg", [TINY, TINY128], ids=["d64", "d128"])
@pytest.mark.parametrize("chunks", [(32, 32, 6), (13, 40, 17)], ids=["32-32-6", "13-40-17"])
def test_joined_gptq_matches_oracle(lib, cuda, cfg, chunks):
    """3 decode rows + a 6- or 13-row chunk run the exact-integer GEMMs (<= 16 rows), 3 + 32 / 40 / 17 the wgmma ones."""
    _scenario(cfg, 5, "f16", 5e-3, chunks, check_kv=True).close()


@pytest.mark.parametrize("dtype,tol", [("f16", 3e-3), ("bf16", 2e-2)])
def test_joined_dense_matches_oracle(lib, cuda, dtype, tol):
    _scenario(TINY, 0, dtype, tol, (32, 32, 6), check_kv=True).close()


def test_joined_awq_matches_oracle(lib, cuda):
    _scenario(TINY, 6, "f16", 5e-3, (32, 32, 6)).close()


# W8A8 turns small attention differences into int8 bucket flips of the next Linear's activations.  At these short
# contexts the decode kernel computes P.V in fp32 and matches the oracle bit for bit; the joined kernel carries P in 11
# bits for fp16 models (as k_decode_attn does at long contexts), ~3e-4 rel on the attention output, which the TINY model
# amplifies to ~2e-2 on the logits.
@pytest.mark.parametrize("dtype,tol", [("f16", 3e-2), ("bf16", 3e-2)])
def test_joined_w8a8_matches_oracle(lib, cuda, dtype, tol):
    _scenario(TINY, 2, dtype, tol, (32, 32, 6)).close()


def test_joined_llama8b_layers_matches_oracle(lib, cuda):
    _scenario(LAYER8B, 5, "f16", 5e-3, (18, 6), sym=True, scale_range=(0.0003, 0.0008), seed=2).close()


def test_joined_step_keeps_device_state(lib, cuda):
    """The device-resident (token, position) state of zl_llama_set_state survives a joined step."""
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=3)
    dec = _decoder(TINY, 5, "f16", sd)
    dec.set_state(np.array([11, 12, 13, 14], np.int32), np.array([7, 8, 9, 10], np.int32))
    before = dec.get_state(4)
    dec.step_joined([(0, np.arange(20, dtype=np.int32), 0, True), (2, np.array([3], np.int32), 5, False)])
    after = dec.get_state(4)
    np.testing.assert_array_equal(before[0], after[0])
    np.testing.assert_array_equal(before[1], after[1])
    dec.close()


SAMPLED = {1: dict(temperature=0.9, top_p=0.9, top_k=50, repetition_penalty=1.3, seed=11),
           3: dict(temperature=1.1, presence_penalty=0.5, seed=7)}


def test_joined_sampling_matches_ops_sample(lib, cuda):
    """A sampled task's pick is ops.sample of its returned logits row with the same parameters, counter = the row's
    position and the task's history; the next step's penalties see that pick."""
    V = TINY["vocab_size"]
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=1)
    dec = _decoder(TINY, 5, "f16", sd)
    pos = np.zeros(4, np.int32)
    for t in range(3):
        dec.prefill(t, np.arange(2 + t, 6 + t, dtype=np.int32))
        pos[t] = 4
    for t, p in SAMPLED.items():
        dec.set_sampling(t, **p)
    params = [dict(temperature=0.0), SAMPLED[1], dict(temperature=0.0), SAMPLED[3]]
    hist = np.zeros((4, (V + 31) // 32), dtype=np.int32)
    prompt = np.arange(100, 130, dtype=np.int32)
    tok = np.array([5, 6, 7], np.int32)
    nxt, logits = dec.step_joined([(t, tok[t:t + 1], int(pos[t]), True) for t in range(3)] + [(3, prompt, 0, True)],
                                  want_logits=True)
    want, hist = _sample(cuda, logits, params, [0, 1, 2, 3], [pos[0], pos[1], pos[2], len(prompt) - 1], hist)
    np.testing.assert_array_equal(nxt, want)
    assert so.bitmap_tokens(hist[3], V) == {int(nxt[3])}
    pos[:3] += 1
    pos[3] = len(prompt)
    for _ in range(3):
        tok = nxt.astype(np.int32)
        nxt, logits = dec.step_joined([(t, tok[t:t + 1], int(pos[t]), True) for t in range(4)], want_logits=True)
        want, hist = _sample(cuda, logits, params, [0, 1, 2, 3], pos, hist)
        np.testing.assert_array_equal(nxt, want)
        pos += 1
    dec.close()


def _raw(dec, tokens, seg):
    """zl_llama_step_joined without the Python-side validation: -> return code"""
    t = np.ascontiguousarray(tokens, dtype=np.int32)
    s = np.ascontiguousarray(seg, dtype=np.int32).reshape(-1, 4)
    nxt = np.empty(max(1, s.shape[0]), np.int32)
    return dec.lib.zl_llama_step_joined(dec.h, t.ctypes.data_as(ctypes.c_void_p), s.ctypes.data_as(ctypes.c_void_p),
                                        s.shape[0], nxt.ctypes.data_as(ctypes.c_void_p), None)


def test_joined_refusals(lib, cuda):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import LlamaDecoder
    INVALID, UNSUPPORTED, STATE = -1, -2, -4
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=4)
    one = [(0, [1], 0, True)]
    dec = _decoder(TINY, 5, "f16", sd, prefill_chunk=0)
    with pytest.raises(_lib.ZLError) as e:
        dec.step_joined(one)
    assert e.value.code == STATE
    dec.close()
    dec = _decoder(TINY, 5, "f16", sd, prefill_chunk=16, kv_cache_dtype="int8")
    with pytest.raises(_lib.ZLError) as e:
        dec.step_joined(one)
    assert e.value.code == UNSUPPORTED
    dec.close()
    tp = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, tp_rank=0, tp_size=2, prefill_chunk=16, **TINY)
    assert _raw(tp, [1], [0, 0, 1, 1]) == UNSUPPORTED
    tp.close()
    dec = _decoder(TINY, 5, "f16", sd, prefill_chunk=16)       # rows <= max(max_batch 4, 16)
    ok = _raw(dec, [1, 2], [[0, 0, 1, 1], [1, 3, 1, 0]])
    assert ok == 0
    for tokens, seg in [([1, 2], [[0, 0, 1, 1], [0, 3, 1, 1]]),      # duplicate task
                        ([1], [4, 0, 1, 1]), ([1], [-1, 0, 1, 1]),    # task out of range
                        ([1], [0, 0, 0, 1]),                          # n < 1
                        ([1], [0, -1, 1, 1]),                         # pos0 < 0
                        ([1, 2], [0, 127, 2, 1]),                     # pos0 + n > max_seq
                        (list(range(17)), [0, 0, 17, 1]),             # too many rows
                        ([1] * 5, [[t, 0, 1, 1] for t in range(5)]),  # nseg > max_batch
                        ([512], [0, 0, 1, 1]), ([-3], [0, 0, 1, 1])]:  # token out of range
        assert _raw(dec, tokens, seg) == INVALID, seg
    # nothing was enqueued by the refused calls: the model still steps
    assert _raw(dec, [1, 2], [[0, 1, 1, 1], [1, 4, 1, 1]]) == 0
    dec.close()
