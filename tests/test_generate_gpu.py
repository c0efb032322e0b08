"""Generate until stop (zl_llama_generate / zl_llama_set_stop) against the host loop: a second LlamaDecoder with the same
weights and prefill, stepped with decode(), the stop rules applied in Python and finished rows fed a dummy position far
past the compared range.  Every model here has max_seq <= 256, so both decoders attend in the one length bucket 256 and
the same inputs give the same bits: tokens, finish reasons and KV rows are compared exactly."""
import ctypes

import numpy as np
import pytest

from oracle import model as omodel
from tests.test_llama_gpu import TINY, TINY128

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED, STATE = -1, -2, -4


def _decoder(cfg, quant, dtype, sd, max_batch=4, max_seq=128, prefill_chunk=32, **kw):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=quant, dtype=dtype, max_batch=max_batch, max_seq=max_seq, prefill_chunk=prefill_chunk,
                       **cfg, **kw)
    dec.load_state_dict(sd)
    return dec


def _prefill(decs, prompts):
    """Prefill every task of every decoder, then set their (token, position) state: -> (tokens, positions)."""
    tok = np.zeros(len(prompts), np.int32)
    pos = np.array([len(p) for p in prompts], np.int32)
    for dec in decs:
        for t, p in enumerate(prompts):
            tok[t] = dec.prefill(t, p)
        dec.set_state(tok, pos)
    return tok, pos


def _host_loop(dec, tok, pos, rules, n_steps, max_seq, dummy):
    """The oracle: n_steps decode() steps of tasks 0 .. b-1 from (tok, pos) with rules[t] = (stop ids, budget) or None
    applied in Python.  -> (emitted token lists, finish reasons, final tokens, final positions)."""
    b = len(tok)
    tok, pos = np.array(tok, np.int32), np.array(pos, np.int32)
    out, fin = [[] for _ in range(b)], np.zeros(b, np.int32)
    for _ in range(n_steps):
        if fin.all():
            break
        live = fin == 0
        nxt = dec.decode(np.where(live, tok, 0), np.where(live, pos, dummy))
        for t in np.nonzero(live)[0]:
            x = int(nxt[t])
            out[t].append(x)
            ids, budget = rules[t] if rules[t] else ((), 0)
            if x in ids:
                fin[t] = 1
            elif budget and len(out[t]) >= budget:
                fin[t] = 2
            elif pos[t] + 1 >= max_seq:
                fin[t] = 3
            tok[t] = x
            pos[t] += 1
    return out, fin, tok, pos


def _set_rules(dec, rules):
    for t, r in enumerate(rules):
        if r:
            dec.set_stop(t, r[0], r[1])


def _first_new(stream, start):
    """A token of the stream that first occurs at index >= start -> (token, index)."""
    for i in range(start, len(stream)):
        if stream[i] not in stream[:i]:
            return stream[i], i
    raise AssertionError("no fresh token in the stream")


def _kv(dec, t, n, layers):
    return [tuple(a.copy() for a in dec.read_kv(l, t, 0, n)) for l in range(layers)]


def _same(a, b):
    return all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for la, lb in zip(a, b) for x, y in zip(la, lb))


PROMPTS = (5, 9, 3, 12)


@pytest.mark.parametrize("cfg,quant,dtype,kv", [(TINY, 5, "f16", None), (TINY128, 5, "f16", None), (TINY, 0, "bf16", None),
                                                (TINY, 5, "f16", "int8")],
                         ids=["gptq-d64", "gptq-d128", "dense-bf16", "gptq-kv8"])
def test_generate_greedy_matches_host_loop(lib, cuda, cfg, quant, dtype, kv):
    sd = omodel.make_state_dict(cfg, quant, 128, False, seed=3, dtype=dtype)
    dec = _decoder(cfg, quant, dtype, sd, kv_cache_dtype=kv)
    ref = _decoder(cfg, quant, dtype, sd, kv_cache_dtype=kv)
    rng = np.random.default_rng(1)
    prompts = [rng.integers(0, cfg["vocab_size"], n).astype(np.int32) for n in PROMPTS]
    tok, pos = _prefill([dec, ref], prompts)
    free, _, _, _ = _host_loop(ref, tok, pos, [None] * 4, 24, 128, 120)
    ref.set_state(tok, pos)
    s0, i0 = _first_new(free[0], 3)
    s2, _ = _first_new(free[2], 6)
    rules = [([s0], 0), ((), 7), ([s2, (s2 + 1) % cfg["vocab_size"]], 20), None]
    want, wfin, _, _ = _host_loop(ref, tok, pos, rules, 24, 128, 120)
    assert wfin[0] == 1 and len(want[0]) == i0 + 1 and wfin[1] == 2 and wfin[3] == 0
    kernels = dec.stats()[1]
    _set_rules(dec, rules)
    got, fin, steps = dec.generate(4, 24)
    assert steps == 24
    for t in range(4):
        assert list(got[t]) == want[t], t
    assert list(fin) == list(wfin)
    assert dec.stats()[1] == kernels                      # the step graphs' count is not the loop's
    # KV rows [0, fed) of every task: the same bits as the host loop's
    gt, gp = dec.get_state(4)
    for t in range(4):
        n = int(PROMPTS[t] + len(want[t]))
        assert gp[t] == n and gt[t] == want[t][-1]        # finished: its last token, at the position it would be fed
        assert _same(_kv(dec, t, n, cfg["num_layers"]), _kv(ref, t, n, cfg["num_layers"])), t
    dec.close()
    ref.close()


def test_generate_staggered_stops(lib, cuda):
    """Tasks stop at different steps, by stop id, budget and the end of a small KV buffer; a finished task emits
    nothing and leaves no trace; a call with every task finished runs no step."""
    MS = 24
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=5)
    dec = _decoder(TINY, 5, "f16", sd, max_seq=MS, prefill_chunk=16)
    ref = _decoder(TINY, 5, "f16", sd, max_seq=MS, prefill_chunk=16)
    rng = np.random.default_rng(2)
    prompts = [rng.integers(0, 512, n).astype(np.int32) for n in (3, 5, 8, 10)]
    tok, pos = _prefill([dec, ref], prompts)
    free, _, _, _ = _host_loop(ref, tok, pos, [None] * 4, 12, MS, MS - 1)
    ref.set_state(tok, pos)
    s1, i1 = _first_new(free[1], 4)
    # 0: budget 20 (runs past 2's end); 1: stop id; 2: no rule, fills the buffer after 16 steps; 3: budget 2
    rules = [((), 20), ([s1], 0), None, ((), 2)]
    want, wfin, wtok, wpos = _host_loop(ref, tok, pos, rules, MS, MS, MS - 1)
    assert list(wfin) == [2, 1, 3, 2] and len(want[2]) == MS - 8 and len(want[0]) == 20
    _set_rules(dec, rules)
    got1, fin1, steps1 = dec.generate(4, 3)               # task 3 stops at step 2
    assert steps1 == 3 and fin1[3] == 2 and list(got1[3]) == want[3]
    snap3 = _kv(dec, 3, 12, 2)
    got2, fin2, steps2 = dec.generate(4, 16 - 3)          # task 2 fills its buffer at the last of these steps
    assert got2[3].size == 0 and fin2[3] == 2             # finished at call start: emits nothing
    assert fin2[2] == 3 and fin2[0] == 0
    snap2 = _kv(dec, 2, MS, 2)
    t2, p2 = dec.get_state(4)
    assert p2[2] == MS and t2[2] == want[2][-1]
    got3, fin3, steps3 = dec.generate(4, MS)              # task 0 runs 4 more steps beside the finished tasks
    assert steps3 == 4 and list(fin3) == list(wfin)
    for t in range(4):
        assert list(got1[t]) + list(got2[t]) + list(got3[t]) == want[t], t
    # no trace: the KV rows of task 2 (the whole buffer: its last row was re-run) and of task 3 up to its last fed row
    assert _same(_kv(dec, 2, MS, 2), snap2)
    assert _same(_kv(dec, 3, 12, 2), snap3)
    t, p = dec.get_state(4)
    assert list(t) == [int(x) for x in wtok] and [int(x) for x in p] == [int(x) for x in wpos]
    # every task finished: 0 steps, nothing enqueued, the state unchanged
    got4, fin4, steps4 = dec.generate(4, 5)
    assert steps4 == 0 and all(g.size == 0 for g in got4) and list(fin4) == list(wfin)
    t4, p4 = dec.get_state(4)
    assert np.array_equal(t4, t) and np.array_equal(p4, p)
    # a task re-armed with a full buffer finishes at once without emitting
    dec.set_stop(2)
    got5, fin5, steps5 = dec.generate(4, 5)
    assert steps5 == 0 and got5[2].size == 0 and fin5[2] == 3
    assert _same(_kv(dec, 2, MS, 2), snap2)
    dec.close()
    ref.close()


def test_generate_chunked_calls(lib, cuda):
    """generate(max_steps=k) called repeatedly gives the tokens of one call, across the length bucket boundary 256."""
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=6)
    one = _decoder(TINY, 5, "f16", sd, max_batch=2, max_seq=320, prefill_chunk=64)
    many = _decoder(TINY, 5, "f16", sd, max_batch=2, max_seq=320, prefill_chunk=64)
    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, 512, n).astype(np.int32) for n in (244, 250)]   # task 1 crosses 256 after 6 steps
    _prefill([one, many], prompts)
    want, fin, steps = one.generate(2, 20)
    assert steps == 20 and list(fin) == [0, 0]
    got = [[], []]
    for k in (3, 3, 3, 3, 3, 3, 2):
        g, f, s = many.generate(2, k)
        assert s == k
        for t in range(2):
            got[t] += list(g[t])
    for t in range(2):
        assert got[t] == list(want[t])
    assert np.array_equal(one.get_state(2)[1], many.get_state(2)[1])
    one.close()
    many.close()


def test_generate_sampling_and_processors(lib, cuda):
    """Sampled tasks, a logit_bias task and an n-gram task emit the host loop's tokens.  A task that finished and sat out
    steps continues, once re-armed, with the tokens of a host loop that never ran the idle steps: its history and
    generated-token sequence were left alone."""
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=7)
    dec = _decoder(TINY, 5, "f16", sd)
    ref = _decoder(TINY, 5, "f16", sd)
    settings = [dict(temperature=0.9, top_p=0.95, seed=11),
                dict(temperature=0.8, top_k=40, repetition_penalty=1.3, seed=5),
                dict(logit_bias={7: 2.5, 100: 1.5, 300: -np.inf}),
                dict(temperature=0.7, ngram_penalty=1.6, seed=9)]
    for d in (dec, ref):
        for t, s in enumerate(settings):
            d.set_sampling(t, **s)
    rng = np.random.default_rng(4)
    prompts = [rng.integers(0, 512, n).astype(np.int32) for n in PROMPTS]
    tok, pos = _prefill([dec, ref], prompts)
    want, _, _, _ = _host_loop(ref, tok, pos, [None] * 4, 22, 128, 120)
    s1, i1 = _first_new(want[1], 3)
    dec.set_stop(1, [s1])
    got1, fin1, steps1 = dec.generate(4, 12)
    assert steps1 == 12 and list(fin1) == [0, 1, 0, 0]
    assert list(got1[1]) == want[1][:i1 + 1]
    dec.set_stop(1)                                        # re-armed after 11 - i1 idle steps
    got2, fin2, steps2 = dec.generate(4, 10)
    assert steps2 == 10 and list(fin2) == [0, 0, 0, 0]
    assert list(got1[1]) + list(got2[1]) == want[1][:i1 + 11]
    for t in (0, 2, 3):
        assert list(got1[t]) + list(got2[t]) == want[t], t
    dec.close()
    ref.close()


def test_generate_continuous_batching(lib, cuda):
    """A prefill of another task between two generate calls leaves the running tasks' tokens unchanged, and the new task
    then joins the batch."""
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=8)
    dec = _decoder(TINY, 5, "f16", sd)
    ref = _decoder(TINY, 5, "f16", sd)
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, 512, n).astype(np.int32) for n in (6, 4, 11)]
    tok, pos = _prefill([ref], prompts)
    want, _, _, _ = _host_loop(ref, tok, pos, [None] * 3, 10, 128, 120)
    _prefill([dec], prompts[:2])
    got1, _, _ = dec.generate(2, 4)
    t3 = dec.prefill(2, prompts[2])
    assert t3 == tok[2]
    got2, _, _ = dec.generate(2, 3)
    t, p = dec.get_state(2)
    dec.set_state(np.append(t, t3), np.append(p, len(prompts[2])))
    got3, _, _ = dec.generate(3, 3)
    for i in range(2):
        assert list(got1[i]) + list(got2[i]) + list(got3[i]) == want[i][:10], i
    assert list(got3[2]) == want[2][:3]
    dec.close()
    ref.close()


def _raw_generate(dec, b, max_steps):
    buf = np.zeros(max(1, b * max_steps), np.int32)
    n = np.zeros(max(1, b), np.int32)
    steps = ctypes.c_int()
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    return dec.lib.zl_llama_generate(dec.h, b, max_steps, p(buf), p(n), p(n), ctypes.byref(steps))


def _raw_stop(dec, task, ids, budget, n=None):
    a = np.array(ids if ids else [0], np.int32)
    return dec.lib.zl_llama_set_stop(dec.h, task, a.ctypes.data_as(ctypes.c_void_p), len(ids) if n is None else n,
                                     budget)


def test_generate_refusals(lib, cuda):
    from zhilight_b200.llama import LlamaDecoder
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=9)
    nograph = _decoder(TINY, 5, "f16", sd, use_graph=False)
    assert _raw_generate(nograph, 1, 1) == UNSUPPORTED
    nograph.decode([1], [0])                                # the model still steps
    nograph.close()
    tp = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, tp_rank=0, tp_size=2, prefill_chunk=16, **TINY)
    assert _raw_generate(tp, 1, 1) == UNSUPPORTED
    assert _raw_stop(tp, 0, [1], 0) == UNSUPPORTED
    tp.close()
    raw = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, **TINY)   # not finalized
    assert _raw_generate(raw, 1, 1) == STATE
    assert _raw_stop(raw, 0, [1], 0) == STATE
    raw.close()
    dec = _decoder(TINY, 5, "f16", sd)
    dec.set_state([1, 2], [0, 0])
    for b, k in [(0, 1), (5, 1), (1, 0), (1, 129), (-1, 4)]:
        assert _raw_generate(dec, b, k) == INVALID, (b, k)
    for task, ids, budget, n in [(-1, [1], 0, None), (4, [1], 0, None), (0, [512], 0, None), (0, [-1], 0, None),
                                 (0, [3, 3], 0, None), (0, list(range(9)), 0, None), (0, [1], -1, None),
                                 (0, [1], 0, -1)]:
        assert _raw_stop(dec, task, ids, budget, n) == INVALID, (task, ids, budget, n)
    # nothing was enqueued or changed by the refused calls: the model still steps, without a stop rule
    got, fin, steps = dec.generate(2, 3)
    assert steps == 3 and list(fin) == [0, 0] and all(g.size == 3 for g in got)
    with pytest.raises(ValueError):
        dec.set_stop(0, [1, 1])
    dec.step_device(2)
    dec.sync()
    dec.close()
