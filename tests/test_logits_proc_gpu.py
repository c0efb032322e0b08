"""Logits processors on the GPU: zl_sample_processed against the numpy contract (tests/ngram_oracle.py), and the decode
driver's picks with a task's n-gram penalty and logit bias on every pick route."""
import ctypes

import numpy as np
import pytest

from oracle import model as omodel
from tests import ngram_oracle as ng
from tests import sampling_oracle as so
from tests.test_llama_gpu import TINY

pytestmark = pytest.mark.gpu

MAXB = 1024


def _t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _device_state(dev, seqs, stride, ngrams, biases, V):
    """device tensors of zl_sample_processed for per-task host state"""
    n = len(seqs)
    seq = np.zeros((n, stride), np.int32)
    for t, s in enumerate(seqs):
        seq[t, :len(s)] = s
    bt = np.zeros((n, MAXB), np.int32)
    bv = np.zeros((n, MAXB), np.float32)
    bc = np.zeros(n, np.int32)
    for t, b in enumerate(biases):
        items = list((b or {}).items())
        bc[t] = len(items)
        for j, (k, v) in enumerate(items):
            bt[t, j], bv[t, j] = k, v
    hist = so.history_bitmap([set(s) for s in seqs], V)
    return dict(seq=_t(seq, dev), seq_len=_t(np.array([len(s) for s in seqs], np.int32), dev),
                ngram_penalty=_t(np.asarray(ngrams, np.float32), dev), bias_tokens=_t(bt, dev), bias_values=_t(bv, dev),
                bias_count=_t(bc, dev), history=_t(hist, dev))


def _run_op(dev, logits, params, seqs, stride, ngrams, biases, row_task=None, counter=None, use_ngram=True):
    """ops.sample_processed on host inputs -> (picks, seq, seq_len, history) as numpy"""
    import torch
    from zhilight_b200 import ops
    V = logits.shape[1]
    st = _device_state(dev, seqs, stride, ngrams, biases, V)
    if not use_ngram:
        st["ngram_penalty"] = None
    rt = None if row_task is None else _t(np.asarray(row_task, np.int32), dev)
    ct = None if counter is None else _t(np.asarray(counter, np.int32), dev)
    out = ops.sample_processed(_t(np.asarray(logits, np.float32), dev), params, st["seq"], st["seq_len"],
                               st["ngram_penalty"], st["bias_tokens"], st["bias_values"], st["bias_count"], rt, ct,
                               st["history"])
    torch.cuda.synchronize()
    return out.cpu().numpy(), st["seq"].cpu().numpy(), st["seq_len"].cpu().numpy(), st["history"].cpu().numpy()


def _lm_rows(rng, n, V):
    l = (rng.normal(size=(n, V)) * 2).astype(np.float32)
    for r in range(n):
        head = rng.choice(V, size=64, replace=False)
        l[r, head] += rng.uniform(8, 16, size=64).astype(np.float32)
    return l


def _slice_tokens(V):
    """the first and last token of each of k_sample's 8 CTA slices (the last one short when 8 does not divide V)"""
    S = -(-V // 8)
    return sorted({t for r in range(8) for t in (r * S, min(V, (r + 1) * S) - 1)})


def _greedy_margin_ok(l):
    top = np.sort(l[np.isfinite(l)])[-2:]
    return top.size < 2 or top[1] - top[0] > 1e-4 * max(1.0, abs(float(top[1])))


# greedy rows: the decisive token ends 0.5 above the row's best (it wins only if its bias is added where and as the
# contract says), 0.5 below it, or 8 above; sampled rows: 8 above (nearly all the mass), level with the best (about half
# the mass) or 0.3 above
DELTA_GREEDY = (0.5, -0.5, 8.0)
DELTA_SAMPLED = (8.0, 0.0, 0.3)


@pytest.mark.parametrize("V", [128256, 152064, 32001])
def test_operator_matches_oracle(lib, cuda, V):
    """Every row has a decisive finite bias on one token: the first or last token of a CTA slice, rotating so that the
    rows cover all 16 (at V = 32001 the last slice is short), and for the 1024-entry row one of its random entries.
    The decisive token's raw logit is 3, so adding its bias, assigning it, or adding it after the temperature all give
    different rows."""
    rng = np.random.default_rng(V)
    edges = _slice_tokens(V)
    n = len(edges) + 1
    stride = 4100
    logits = _lm_rows(rng, n, V)
    logits[:, edges] = 3.0
    heads = [np.argsort(-logits[r])[:40] for r in range(n)]
    seqs = []
    for t in range(n):
        kind = t % 4
        if kind == 0:      # text-like: the row's head tokens in random order
            seqs.append(rng.choice(heads[t], size=int(rng.integers(1, 1200))).tolist())
        elif kind == 1:    # one repeated token
            seqs.append([int(heads[t][0])] * (4096 if t == 1 else 700))
        elif kind == 2:    # a loop of period 2-7
            p = int(rng.integers(2, 8))
            seqs.append([int(heads[t][k % p]) for k in range(4096 if t == 2 else 1500)])
        else:              # a loop after a text-like prefix
            seqs.append(rng.choice(heads[t], size=300).tolist() + [int(h) for h in heads[t][:5]] * 50)
    ngrams = [1.0 if t in (3, 9) else 1.3 for t in range(n)]
    params = []
    for t in range(n):
        if t % 3 == 0:
            params.append(dict(temperature=0.0, repetition_penalty=1.1))
        else:
            params.append(dict(temperature=float(rng.choice([0.7, 1.0])), top_p=float(rng.choice([1.0, 0.95])),
                               top_k=int(rng.choice([0, 50])), repetition_penalty=1.1,
                               seed=int(rng.integers(0, 2 ** 63))))
    biases, decisive = [], []
    for t in range(n):
        b = {int(k): float(rng.uniform(-3, 3)) for k in edges}
        b[int(heads[t][1])] = float("-inf")                    # bans a token
        if t == 5:   # 1024 entries, one of the random ones decisive
            extra = rng.choice(np.setdiff1d(np.arange(V), np.concatenate([list(b), heads[t]])), size=MAXB - len(b),
                               replace=False)
            b.update({int(k): float(rng.uniform(-4, 4)) for k in extra})
            logits[t, extra] = 3.0
            d = int(extra[17])
        else:
            d = edges[(t if t < 5 else t - 1) % len(edges)]
        del b[d]
        with np.errstate(over="ignore"):
            best = float(np.max(ng.process(logits[t], seqs[t], params[t]["repetition_penalty"], 0.0, ngrams[t], b)))
        greedy = so.is_greedy(params[t]["temperature"], params[t].get("top_k", 0))
        delta = (DELTA_GREEDY if greedy else DELTA_SAMPLED)[(t // 3) % 3]
        b[d] = float(np.float32(best - 3.0 + delta))
        biases.append(b)
        decisive.append((d, delta))
    assert {d for d, _ in decisive} >= set(edges)
    row_task = rng.permutation(n)           # row i holds task row_task[i]
    row_logits = logits[row_task]
    counter = rng.integers(0, 2 ** 20, size=n)
    got, seq, seq_len, hist = _run_op(cuda, row_logits, params, seqs, stride, ngrams, biases, row_task, counter)
    amb = decided = 0
    with np.errstate(over="ignore"):
        for i in range(n):
            t = int(row_task[i])
            l = ng.process(row_logits[i], seqs[t], params[t]["repetition_penalty"], 0.0, ngrams[t], biases[t])
            want, ambiguous = ng.pick(row_logits[i], seqs[t], params[t], counter[i], ngrams[t], biases[t])
            assert got[i] != int(heads[t][1])   # -inf bias
            greedy = so.is_greedy(params[t]["temperature"], params[t].get("top_k", 0))
            if ambiguous or (greedy and not _greedy_margin_ok(l)):
                amb += 1
                continue
            assert got[i] == want, (i, t, got[i], want, decisive[t])
            decided += want == decisive[t][0]
            # the pick is appended to the task's sequence and set in its history
            assert seq_len[t] == len(seqs[t]) + 1 and seq[t, len(seqs[t])] == got[i]
            assert int(got[i]) in so.bitmap_tokens(hist[t], V)
    assert amb <= 1
    assert decided >= n // 3   # the biased token decides many rows


def test_ngram_beyond_shared_memory_and_capacity(lib, cuda):
    """sequences longer than k_ngram_levels' shared-memory stage, empty and one-token sequences, and a full sequence
    (the append is dropped)"""
    rng = np.random.default_rng(5)
    V, stride = 1000, 16000
    logits = _lm_rows(rng, 5, V)
    loop = [int(x) for x in np.argsort(-logits[0])[:5]]
    seqs = [rng.choice(np.argsort(-logits[0])[:30], size=15000).tolist() + loop * 100,
            [int(np.argmax(logits[1]))] * 13000,
            [], [int(np.argmax(logits[3]))],
            (loop * 3200)[:stride]]
    params = [dict(temperature=0.0, repetition_penalty=1.05)] * 5
    ngrams = [1.02] * 5
    got, seq, seq_len, _ = _run_op(cuda, logits, params, seqs, stride, ngrams, [None] * 5)
    with np.errstate(over="ignore"):
        for t in range(5):
            l = ng.process(logits[t], seqs[t], 1.05, 0.0, ngrams[t])
            if _greedy_margin_ok(l):
                assert got[t] == so.greedy(l), t
    assert seq_len.tolist() == [len(s) + 1 for s in seqs[:4]] + [stride]
    np.testing.assert_array_equal(seq[4], seqs[4])


def test_rows_without_processors_match_zl_sample(lib, cuda):
    """tasks with no bias and ngram <= 1 pick exactly what zl_sample picks, with or without the n-gram launch"""
    import torch
    from zhilight_b200 import ops
    rng = np.random.default_rng(11)
    n, V = 16, 128256
    logits = _lm_rows(rng, n, V)
    seqs = [rng.integers(0, V, size=int(rng.integers(0, 50))).tolist() for _ in range(n)]
    params = [dict(temperature=0.9, top_p=0.9, repetition_penalty=1.2, presence_penalty=0.3 * (t % 2), seed=t)
              if t % 4 else dict(temperature=0.0, repetition_penalty=1.2) for t in range(n)]
    counter = np.arange(n) * 7
    h = _t(so.history_bitmap([set(s) for s in seqs], V), cuda)
    want = ops.sample(_t(logits, cuda), params, None, _t(counter.astype(np.int32), cuda), h).cpu().numpy()
    torch.cuda.synchronize()
    for use_ngram in (True, False):
        got, _, _, _ = _run_op(cuda, logits, params, seqs, 64, [1.0] * n, [None] * n, None, counter, use_ngram)
        np.testing.assert_array_equal(got, want)


# ------------------------------------------------------------------------------------------ decode driver
V_TINY = TINY["vocab_size"]
BIAS = {0: 1.5, 63: -1.0, 64: 0.5, 200: 2.0, 300: -np.inf, 447: 0.25, 448: 1.0, V_TINY - 1: 3.0}


def _settings(sampled, others):
    p0 = (dict(temperature=0.8, top_p=0.95, repetition_penalty=1.1, seed=17) if sampled
          else dict(temperature=0.0, repetition_penalty=1.1))
    s = {0: (p0, 1.3, BIAS)}
    if others == "plain":
        s.update({t: ({}, 1.0, None) for t in (1, 2, 3)})
    else:
        s.update({1: ({}, 1.0, None), 2: (dict(temperature=1.0, seed=3), 1.0, {7: 4.0}),
                  3: (dict(temperature=0.0, repetition_penalty=1.2), 1.5, None)})
    return s


def _want(cuda, logits, s, seqs, tasks, counters):
    """picks of ops.sample_processed for rows of `tasks` over the driver's raw logits, each also checked against the numpy
    oracle where the pick is not within rounding of a boundary; appends them to seqs"""
    n = len(seqs)
    params = [s[t][0] for t in range(n)]
    got, _, _, _ = _run_op(cuda, logits, params, seqs, 256, [s[t][1] for t in range(n)], [s[t][2] for t in range(n)],
                           tasks, counters)
    for r, (t, g) in enumerate(zip(tasks, got)):
        p = dict(dict(temperature=0.0, repetition_penalty=1.0), **params[t])
        with np.errstate(over="ignore"):
            l = ng.process(logits[r], seqs[t], p["repetition_penalty"], p.get("presence_penalty", 0.0), s[t][1], s[t][2])
        want, ambiguous = ng.pick(logits[r], seqs[t], p, counters[r], s[t][1], s[t][2])
        if not ambiguous and (not so.is_greedy(p["temperature"], p.get("top_k", 0)) or _greedy_margin_ok(l)):
            assert g == want, (t, g, want)
        seqs[t].append(int(g))
    return got


def _drive(cuda, sd, quant, kv, mode, sampled, others="mixed", steps=64):
    """4 tasks (1 with others="alone"); task 0 prefilled and then stepped with processors.  Every pick must equal the operator on the step's raw
    logits with each task's own sequence.  Returns task 0's tokens and the (tokens, positions, logits) of its steps."""
    from zhilight_b200.llama import LlamaDecoder
    B = 1 if others == "alone" else 4
    dec = LlamaDecoder(quant_type=quant, dtype="f16", max_batch=B, max_seq=128, prefill_chunk=16, kv_cache_dtype=kv, **TINY)
    dec.load_state_dict(sd)
    s = {t: v for t, v in _settings(sampled, others).items() if t < B}
    for t, (p, ngp, b) in s.items():
        dec.set_sampling(t, **p, ngram_penalty=ngp, logit_bias=b)
    seqs = [[] for _ in range(B)]
    prompt = np.array([5, 9, 5, 9, 5, 9, 11], np.int32)
    t0, l0 = dec.prefill(0, prompt, want_logits=True)
    assert t0 == _want(cuda, l0, s, seqs, [0], [len(prompt) - 1])[0]
    tok = np.array([t0, 1, 2, 3][:B], np.int32)
    pos = np.array([len(prompt), 0, 0, 0][:B], np.int32)
    trace = []
    if mode == "device":
        dec.set_state(tok, pos)
    for _ in range(steps):
        if mode == "host":
            nxt, logits = dec.decode(tok, pos, want_logits=True)
        elif mode == "device":
            dec.step_device(B)
            nxt, npos = dec.get_state(B)
            np.testing.assert_array_equal(npos, pos + 1)
            logits = dec.get_logits(B)
        else:
            nxt, logits = dec.step_joined([(t, tok[t:t + 1], int(pos[t]), True) for t in range(B)], want_logits=True)
        want = _want(cuda, logits, s, seqs, list(range(B)), pos)
        np.testing.assert_array_equal(nxt, want)
        if B > 1:
            assert nxt[1] == int(np.argmax(logits[1]))
        trace.append((tok.copy(), pos.copy(), logits.copy()))
        tok, pos = np.asarray(nxt, np.int32), pos + 1
    dec.close()
    return np.array(seqs[0]), trace


@pytest.mark.parametrize("quant,kv", [(5, None), (5, "int8"), (0, None), (0, "int8")],
                         ids=["gptq", "gptq-kv8", "dense", "dense-kv8"])
@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
def test_driver_picks_match_operator(lib, cuda, quant, kv, sampled):
    sd = omodel.make_state_dict(TINY, quant, 128, False, seed=4, dtype="f16")
    host, _ = _drive(cuda, sd, quant, kv, "host", sampled)
    dev, _ = _drive(cuda, sd, quant, kv, "device", sampled)
    np.testing.assert_array_equal(host, dev)
    if kv is None:
        # joined steps (activation-dtype cache only) attend through zl_varlen_attention, whose logits differ from the
        # decode kernels' in the last bits, so only each of their picks is checked against the operator
        _drive(cuda, sd, quant, kv, "joined", sampled)
    # the batch's other tasks (plain, or with their own processors and sampling) do not change task 0's tokens
    plain, _ = _drive(cuda, sd, quant, kv, "host", sampled, others="plain")
    np.testing.assert_array_equal(host, plain)
    alone, _ = _drive(cuda, sd, quant, kv, "host", sampled, others="alone")
    np.testing.assert_array_equal(host, alone)


def test_driver_returns_raw_logits(lib, cuda):
    """want_logits returns the lm_head output: a decoder without processors fed the same tokens returns the same rows"""
    from zhilight_b200.llama import LlamaDecoder
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=4, dtype="f16")
    _, trace = _drive(cuda, sd, 5, None, "host", True, steps=8)
    dec = LlamaDecoder(quant_type=5, dtype="f16", max_batch=4, max_seq=128, prefill_chunk=16, **TINY)
    dec.load_state_dict(sd)
    dec.prefill(0, np.array([5, 9, 5, 9, 5, 9, 11], np.int32))
    for tok, pos, logits in trace:
        _, plain = dec.decode(tok, pos, want_logits=True)
        np.testing.assert_array_equal(plain, logits)
    dec.close()


def test_kernels_per_step(lib, cuda):
    """no processor task: the launches of plain sampling / greedy; bias adds none; the n-gram rule adds one"""
    from zhilight_b200.llama import LlamaDecoder
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=2)
    counts = {}
    for setup, kw in (("greedy", dict()), ("sampled", dict(temperature=0.7, seed=3)),
                      ("off", dict(temperature=0.7, seed=3, ngram_penalty=1.0, logit_bias={})),
                      ("bias", dict(temperature=0.7, seed=3, logit_bias={4: 1.0})),
                      ("greedy_bias", dict(logit_bias={4: 1.0})),
                      ("ngram", dict(temperature=0.7, seed=3, ngram_penalty=1.2))):
        dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, **TINY)
        dec.load_state_dict(sd)
        dec.set_sampling(1, **kw)
        dec.decode(np.array([1, 2], np.int32), np.array([0, 0], np.int32))
        counts[setup] = dec.stats(2)[1]
        dec.close()
    assert counts["off"] == counts["sampled"] == counts["bias"] == counts["greedy_bias"] == counts["greedy"] - 1
    assert counts["ngram"] == counts["sampled"] + 1


def _set_proc(dec, task, ngram, toks, vals, n=None):
    t = np.ascontiguousarray(toks, np.int32)
    v = np.ascontiguousarray(vals, np.float32)
    return dec.lib.zl_llama_set_logits_processors(dec.h, task, ctypes.c_float(ngram), t.ctypes.data_as(ctypes.c_void_p),
                                                  v.ctypes.data_as(ctypes.c_void_p), t.size if n is None else n)


def test_refusals_enqueue_nothing(lib, cuda):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import LlamaDecoder
    tp = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, tp_rank=0, tp_size=2, **TINY)
    assert _set_proc(tp, 0, 1.0, [3], [1.0]) == -2
    assert _set_proc(tp, 0, 1.3, [], []) == -2
    # LlamaDecoder.set_sampling refuses before either C call, so neither the sampling nor the processors change
    for kw in (dict(logit_bias={3: 1.0}), dict(ngram_penalty=1.3)):
        with pytest.raises(_lib.ZLError) as e:
            tp.set_sampling(0, temperature=0.0, **kw)
        assert e.value.code == -2
    tp.close()

    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=6, dtype="f16")
    dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=64, **TINY)
    dec.load_state_dict(sd)
    V = V_TINY
    bad = [(1.0, [3, 3], [1.0, 2.0]), (1.0, [-1], [1.0]), (1.0, [V], [1.0]), (1.0, [3], [np.nan]), (1.0, [3], [np.inf]),
           (1.0, list(range(1025)), [0.0] * 1025), (0.0, [], []), (np.nan, [], []), (np.inf, [], []), (-1.0, [], [])]
    for ngp, toks, vals in bad:
        assert _set_proc(dec, 0, ngp, toks, vals) == -1, (ngp, toks[:3], vals[:3])
    assert _set_proc(dec, 5, 1.0, [], []) == -1
    # nothing was enqueued: the tasks are still plain greedy
    tok, pos = np.array([1, 2], np.int32), np.array([0, 0], np.int32)
    for _ in range(3):
        nxt, logits = dec.decode(tok, pos, want_logits=True)
        np.testing.assert_array_equal(nxt, np.argmax(logits, axis=1))
        tok, pos = nxt, pos + 1
    # a beam step over a task with processors is refused, and runs once they are off
    dec.set_sampling(0, logit_bias={7: -np.inf})
    with pytest.raises(_lib.ZLError) as e:
        dec.beam_step(tok, pos, [[0, 2]], [0.0, 0.0], 2)
    assert e.value.code == -4
    dec.set_sampling(0)
    dec.beam_step(tok, pos, [[0, 2]], [0.0, 0.0], 2)
    dec.close()
