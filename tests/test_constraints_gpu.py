"""Constrained decoding on the GPU: zl_sample_masked against the numpy contract (tests/constraint_oracle.py), and the decode
driver's token automata on every pick route (decode, prefill, joined steps, generate), with their refusals."""
import os
import types

import numpy as np
import pytest

from oracle import model as omodel
from tests import constraint_oracle as co
from tests.test_generate_gpu import _host_loop
from tests.test_llama_gpu import LAYER8B, TINY
from tests.test_logits_proc_gpu import _device_state, _lm_rows, _t
from zhilight_b200 import constraints as C

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED, STATE = -1, -2, -4


# ------------------------------------------------------------------------------------------------------------------
# the operator
# ------------------------------------------------------------------------------------------------------------------

def _op_state(dev, seqs, ngrams, biases, V):
    return _device_state(dev, seqs, 4100, ngrams, biases, V)


def _masked(dev, logits, params, masks, mask_row, seqs, ngrams, biases, row_task, counter):
    import torch
    from zhilight_b200 import ops
    V = logits.shape[1]
    st = _op_state(dev, seqs, ngrams, biases, V)
    out = ops.sample_masked(_t(logits, dev), params, _t(masks.view(np.int32), dev), _t(mask_row, dev), st["seq"],
                            st["seq_len"], st["ngram_penalty"], st["bias_tokens"], st["bias_values"], st["bias_count"],
                            _t(row_task, dev), _t(counter, dev), st["history"])
    torch.cuda.synchronize()
    return out.cpu().numpy(), st["seq_len"].cpu().numpy()


def _processed(dev, logits, params, seqs, ngrams, biases, row_task, counter):
    import torch
    from zhilight_b200 import ops
    V = logits.shape[1]
    st = _op_state(dev, seqs, ngrams, biases, V)
    out = ops.sample_processed(_t(logits, dev), params, st["seq"], st["seq_len"], st["ngram_penalty"], st["bias_tokens"],
                               st["bias_values"], st["bias_count"], _t(row_task, dev), _t(counter, dev), st["history"])
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _operator_case(V, seed):
    """Tasks 0-17 are masked (1, 10 or V/2 allowed tokens; greedy or sampled; with or without bias, -inf bias,
    repetition penalty or the n-gram rule); tasks 18-21 are not; task 22 has every allowed token banned by its bias."""
    rng = np.random.default_rng(seed)
    n = 23
    logits = _lm_rows(rng, n, V)
    logits[3, rng.choice(V, 5)] = np.nan
    masks = np.zeros((n, C.mask_words(V)), np.uint32)
    mask_row = np.arange(n, dtype=np.int32)
    params, seqs, ngrams, biases = [], [], [], []
    for t in range(n):
        size = (1, 10, V // 2)[t % 3]
        if t in (1, 4, 7):   # the masked set holds the row's head tokens: the mask decides within the likely ones
            allowed = np.argsort(-logits[t])[:size] if size < V // 2 else rng.choice(V, size, replace=False)
        else:
            allowed = rng.choice(V, size, replace=False)
        allowed = np.append(allowed, [V - 1] if t == 5 else [])   # the last token, in the tail word at V = 1000
        masks[t] = C.token_bitmask(allowed.astype(np.int64), V)
        sampled = (t // 3) % 2 == 1
        p = dict(temperature=0.0)
        if sampled:
            p = dict(temperature=float(rng.choice([0.7, 1.0])), top_p=float(rng.choice([1.0, 0.9])),
                     top_k=int(rng.choice([0, 3, 50])), seed=int(rng.integers(0, 2 ** 63)))
        heads = np.argsort(-logits[t])[:30]
        seq = rng.choice(heads, size=int(rng.integers(0, 60))).tolist()
        kind = t % 4
        if kind == 1:
            p["repetition_penalty"] = 1.3
        ngram = 1.4 if kind == 2 and seq else 1.0
        b = {}
        if kind in (0, 3):
            al = C.bitmask_tokens(masks[t])
            b = {int(k): float(rng.uniform(-3, 3)) for k in rng.choice(al, min(4, al.size), replace=False)}
            b[int(heads[0])] = float("-inf")
            b.setdefault(int(rng.integers(0, V)), 5.0)   # most likely a masked token: the bias does not unmask it
        params.append(p)
        seqs.append(seq)
        ngrams.append(ngram)
        biases.append(b)
    mask_row[18:22] = -1
    banned = C.bitmask_tokens(masks[22])
    biases[22] = {int(k): float("-inf") for k in banned}
    params[22] = dict(temperature=0.9, seed=5)
    row_task = rng.permutation(n).astype(np.int32)
    counter = rng.integers(0, 2 ** 20, size=n).astype(np.int32)
    return logits[row_task], params, masks, mask_row, seqs, ngrams, biases, row_task, counter


@pytest.mark.parametrize("V", [1000, 128256])
def test_operator_matches_oracle(lib, cuda, V):
    logits, params, masks, mask_row, seqs, ngrams, biases, row_task, counter = _operator_case(V, V)
    got, seq_len = _masked(cuda, logits, params, masks, mask_row, seqs, ngrams, biases, row_task, counter)
    again, _ = _masked(cuda, logits, params, masks, mask_row, seqs, ngrams, biases, row_task, counter)
    assert np.array_equal(got, again)                       # a launch reproduces bit for bit
    plain = _processed(cuda, logits, params, seqs, ngrams, biases, row_task, counter)
    amb = 0
    for i, t in enumerate(row_task):
        if mask_row[t] < 0:
            assert got[i] == plain[i], (i, t)                # unmasked rows: zl_sample_processed's token
            continue
        allowed = C.bitmask_tokens(masks[t])
        assert got[i] in set(allowed.tolist()), (i, t)
        want, ambiguous = co.masked_pick(logits[i], allowed, seqs[t], params[t], counter[i], ngrams[t], biases[t])
        if ambiguous:
            amb += 1
            continue
        assert got[i] == want, (i, t, got[i], want)
        assert seq_len[t] == len(seqs[t]) + 1
    assert amb <= 1
    t22 = int(np.flatnonzero(row_task == 22)[0])
    assert got[t22] == C.bitmask_tokens(masks[22])[0]       # every allowed token banned: the smallest allowed


def test_operator_without_mask_row(lib, cuda):
    """mask_row NULL masks task t by row t; a greedy one-token mask picks that token whatever the logits."""
    import torch
    from zhilight_b200 import ops
    V = 1000
    rng = np.random.default_rng(3)
    logits = _lm_rows(rng, 4, V)
    toks = [0, 999, 31, 32]
    masks = np.stack([C.token_bitmask([x], V) for x in toks])
    out = ops.sample_masked(_t(logits, cuda), dict(temperature=0.0), _t(masks.view(np.int32), cuda))
    torch.cuda.synchronize()
    assert out.cpu().tolist() == toks


# ------------------------------------------------------------------------------------------------------------------
# the decode driver
# ------------------------------------------------------------------------------------------------------------------

def _decoder(cfg, sd, max_batch=4, max_seq=128, prefill_chunk=16, sym=False, states=64, edges=64, **kw):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=5, sym=sym, max_batch=max_batch, max_seq=max_seq, prefill_chunk=prefill_chunk, **cfg,
                       **kw)
    dec.load_state_dict(sd)
    if states:
        dec.enable_constraints(states, edges)
    return dec


MODELS = {"tiny": (TINY, dict(sym=False), None), "layer8b": (LAYER8B, dict(sym=True), (0.0003, 0.0008))}


def _model(name, seed=7):
    cfg, kw, scales = MODELS[name]
    return cfg, kw, omodel.make_state_dict(cfg, 5, 128, kw["sym"], seed=seed, scale_range=scales)


def _choices(V):
    """A trie whose root has 38 children (the kernel binary-searches them), with prefix choices and shared prefixes."""
    rng = np.random.default_rng(V)
    x = [int(v) for v in rng.choice(np.arange(3, V), 48, replace=False)]
    a, b, c, d = x[:4]
    seqs = [[a, b, c], [a, d], [c], [a]] + [[v] for v in x[4:36]] + [[x[36 + i], x[40 + i], x[44 + i]] for i in range(4)]
    return C.choices(seqs, [1, 2], V), seqs


@pytest.mark.parametrize("model", ["tiny", "layer8b"])
@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
def test_generate_emits_one_choice(lib, cuda, model, sampled):
    """Tasks 0-2 answer with one choice of the trie, then an end id (their stop ids); task 3 is unconstrained.  The
    prefill's pick is the first token of the answer.  generate agrees with a host loop of decode steps, the tokens spell
    a choice, constraint_state follows the trie, and task 3 emits what it emits in a decoder without constraints."""
    cfg, kw, sd = _model(model)
    V = cfg["vocab_size"]
    aut, seqs = _choices(V)
    dec, ref = _decoder(cfg, sd, **kw), _decoder(cfg, sd, **kw)
    plain = _decoder(cfg, sd, states=0, **kw)
    rng = np.random.default_rng(1)
    prompts = [rng.integers(0, V, n).astype(np.int32) for n in (5, 20, 3, 9)]
    rules = [([1, 2], 0)] * 3 + [((), 12)]
    first = {}
    for d in (dec, ref, plain):
        for t in range(4):
            if sampled:
                d.set_sampling(t, temperature=1.0, top_k=(0, 3, 50, 0)[t], seed=100 + t)
            if t < 3 and d is not plain:
                d.set_constraint(t, aut)
        tok = np.array([d.prefill(t, p) for t, p in enumerate(prompts)], np.int32)
        first[id(d)] = tok
        d.set_state(tok, np.array([len(p) for p in prompts], np.int32))
    assert np.array_equal(first[id(dec)], first[id(ref)])
    for t, r in enumerate(rules):
        dec.set_stop(t, r[0], r[1])
        plain.set_stop(t, r[0], r[1])
    got, fin, _ = dec.generate(4, 40)
    want, wfin, _, _ = _host_loop(ref, first[id(ref)], [len(p) for p in prompts], rules, 40, 128, 120)
    pgot, _, _ = plain.generate(4, 40)
    states = dec.constraint_state(4)
    for t in range(3):
        assert list(got[t]) == want[t], t
        answer = [int(first[id(dec)][t])] + list(got[t])
        assert fin[t] == 1 and answer[-1] in (1, 2), answer
        assert answer[:-1] in seqs, answer
        assert states[t] == co.run_automaton(aut, answer)[-1] == aut.n_states - 1
    assert states[3] == -1
    assert list(got[3]) == want[3] == list(pgot[3])
    assert first[id(dec)][3] == first[id(plain)][3]
    for d in (dec, ref, plain):
        d.close()


def test_decode_per_step_masks(lib, cuda):
    """A host grammar engine's loop: a fresh one-state mask before every decode step.  Greedy and sampled picks equal
    the masked oracle's on the returned (raw) logits; the mask of a finished step does not leak into the next."""
    cfg, kw, sd = _model("tiny", seed=3)
    V = cfg["vocab_size"]
    dec = _decoder(cfg, sd, **kw)
    params = [dict(temperature=0.0), dict(temperature=0.8, seed=4), dict(temperature=1.0, top_k=5, seed=9),
              dict(temperature=0.0)]
    for t, p in enumerate(params):
        dec.set_sampling(t, **p)
    dec.set_sampling(3, logit_bias={7: 3.0, 11: -np.inf})
    rng = np.random.default_rng(0)
    tok = rng.integers(0, V, 4).astype(np.int32)
    amb = 0
    for pos in range(12):
        masks = []
        for t in range(4):
            m = C.token_bitmask(rng.choice(V, (1, 10, V // 2)[(t + pos) % 3], replace=False), V)
            masks.append(m)
            dec.set_constraint(t, C.allowed(bitmask=m, vocab_size=V))
        nxt, logits = dec.decode(tok, np.full(4, pos, np.int32), want_logits=True)
        for t in range(4):
            bias = {7: 3.0, 11: -np.inf} if t == 3 else None
            want, ambiguous = co.masked_pick(logits[t], C.bitmask_tokens(masks[t]), (), params[t], pos, bias=bias)
            assert nxt[t] in set(C.bitmask_tokens(masks[t]).tolist())
            if ambiguous:
                amb += 1
                continue
            assert nxt[t] == want, (pos, t)
        assert list(dec.constraint_state(4)) == [0] * 4
        tok = nxt
    assert amb <= 1
    dec.close()


def test_states_follow_the_trie_each_step(lib, cuda):
    """Host decode steps over the 38-child trie: after every step each task's state is the trie's next state of its
    pick, and the picks spread over many of the root's edges (the kernel's edge search, not only its default)."""
    cfg, kw, sd = _model("tiny", seed=9)
    V = cfg["vocab_size"]
    aut, _ = _choices(V)
    dec = _decoder(cfg, sd, **kw)
    roots = set()
    for rnd in range(4):
        for t in range(4):
            dec.set_sampling(t, temperature=3.0, seed=17 * rnd + t)
            dec.set_constraint(t, aut)
        prev = dec.constraint_state(4)
        tok = np.array([5, 9, 3, 12], np.int32)
        for pos in range(5):
            nxt = dec.decode(tok, np.full(4, pos, np.int32))
            st = dec.constraint_state(4)
            for t in range(4):
                assert int(nxt[t]) in set(aut.allowed_tokens(int(prev[t])).tolist()), (rnd, pos, t)
                assert st[t] == aut.next_state(int(prev[t]), int(nxt[t])), (rnd, pos, t)
                if prev[t] == aut.start:
                    roots.add(int(nxt[t]))
            prev, tok = st, nxt
    assert len(roots) >= 6, roots
    dec.close()


def test_prefill_and_joined_rows(lib, cuda):
    """The last prefill chunk picks from the start state and moves it once (the other chunks pick nothing); in a joined
    step the emitting segments pick from their states and move, a non-emitting prompt chunk leaves its task's state."""
    cfg, kw, sd = _model("tiny", seed=5)
    V = cfg["vocab_size"]
    aut, _ = _choices(V)
    dec = _decoder(cfg, sd, **kw)
    for t in range(4):
        dec.set_constraint(t, aut)
    rng = np.random.default_rng(2)
    prompt = rng.integers(0, V, 40).astype(np.int32)        # three chunks of 16
    x0, lg = dec.prefill(0, prompt, want_logits=True)
    assert x0 == co.masked_pick(lg[0], aut.allowed_tokens(aut.start))[0]
    assert dec.constraint_state(4)[0] == aut.next_state(aut.start, x0)
    x1 = dec.prefill(1, prompt[:7])
    st = dec.constraint_state(4)
    segs = [(0, [x0], 40, True), (1, [x1], 7, True), (2, rng.integers(0, V, 10).astype(np.int32), 0, False),
            (3, rng.integers(0, V, 4).astype(np.int32), 0, True)]
    nxt, logits = dec.step_joined(segs, want_logits=True)
    after = dec.constraint_state(4)
    for row, (t, s) in enumerate([(0, st[0]), (1, st[1]), (3, st[3])]):
        assert nxt[t] == co.masked_pick(logits[row], aut.allowed_tokens(s))[0], t
        assert after[t] == aut.next_state(s, int(nxt[t])), t
    assert nxt[2] == -1 and after[2] == aut.start
    dec.close()


def _raw_set(dec, task, n_states, masks, row_ptr, edge_tok, edge_next, default_next, start):
    from zhilight_b200 import _lib
    a = types.SimpleNamespace(vocab_size=dec.cfg.vocab_size, n_states=n_states, n_edges=np.asarray(edge_tok).size,
                              masks=np.ascontiguousarray(masks, np.uint32), row_ptr=np.asarray(row_ptr, np.int32),
                              edge_tok=np.asarray(edge_tok, np.int32), edge_next=np.asarray(edge_next, np.int32),
                              default_next=np.asarray(default_next, np.int32), start=start)
    try:
        dec.set_constraint(task, a)
    except _lib.ZLError as e:
        return e.code
    return 0


def test_refusals_enqueue_nothing(lib, cuda):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import LlamaDecoder
    cfg, kw, sd = _model("tiny", seed=6)
    V = cfg["vocab_size"]
    dec = _decoder(cfg, sd, states=0, **kw)
    aut, _ = _choices(V)
    with pytest.raises(_lib.ZLError) as e:                  # not enabled
        dec.set_constraint(0, aut)
    assert e.value.code == STATE
    with pytest.raises(_lib.ZLError) as e:
        dec.constraint_state(2)
    assert e.value.code == STATE
    for s, ed in ((0, 4), (4, -1)):
        with pytest.raises(_lib.ZLError) as e:
            dec.enable_constraints(s, ed)
        assert e.value.code == INVALID
    dec.enable_constraints(aut.n_states, aut.n_edges)
    with pytest.raises(_lib.ZLError) as e:
        dec.enable_constraints(4, 4)
    assert e.value.code == STATE
    small = C.allowed([5], V)
    with pytest.raises(_lib.ZLError) as e:                  # task out of range
        dec.set_constraint(4, small)
    assert e.value.code == INVALID
    # the caps, and malformed automata the Python class would refuse
    big = C.choices([list(range(3, 3 + aut.n_states))], [1], V)
    assert _raw_set(dec, 0, big.n_states, big.masks, big.row_ptr, big.edge_tok, big.edge_next, big.default_next, 0) \
        == INVALID
    m = small.masks
    for args in [(1, m * 0, [0, 0], [], [], [0], 0),                       # empty mask
                 (1, m, [0, 1], [6], [0], [0], 0),                         # edge token outside the mask
                 (1, m, [0, 0], [], [], [1], 0),                           # default out of range
                 (1, m, [0, 0], [], [], [0], 1)]:                          # start out of range
        assert _raw_set(dec, 0, *args) == INVALID, args
    # a constrained task refuses beam steps
    dec.set_constraint(1, small)
    with pytest.raises(_lib.ZLError) as e:
        dec.beam_step([1, 2], [0, 0], [[0, 2]], [0.0, 0.0], 2)
    assert e.value.code == STATE
    dec.set_constraint(1, None)
    # nothing was enqueued by the refused calls: task 0 is unconstrained and decodes as a plain decoder does
    assert list(dec.constraint_state(2)) == [-1, -1]
    plain = _decoder(cfg, sd, states=0, **kw)
    tok = np.array([3, 9], np.int32)
    for pos in range(4):
        a, b = dec.decode(tok, np.full(2, pos, np.int32)), plain.decode(tok, np.full(2, pos, np.int32))
        assert np.array_equal(a, b)
        tok = a
    dec.close()
    plain.close()
    # tensor parallelism without the vocabulary gather: an automaton is refused before anything else
    tp = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, tp_rank=0, tp_size=2, **TINY)
    with pytest.raises(_lib.ZLError) as e:
        tp.set_constraint(0, small)
    assert e.value.code == UNSUPPORTED
    tp.close()


def test_set_sampling_leaves_the_constraint(lib, cuda):
    cfg, kw, sd = _model("tiny", seed=8)
    V = cfg["vocab_size"]
    dec = _decoder(cfg, sd, **kw)
    dec.set_constraint(0, C.allowed([77], V))
    dec.set_sampling(0, temperature=1.0, seed=3)
    dec.set_sampling(0)
    nxt = dec.decode([1, 2], [0, 0])
    assert nxt[0] == 77 and list(dec.constraint_state(2)) == [0, -1]
    dec.close()


# ------------------------------------------------------------------------------------------------------------------
# tensor parallelism: two ranks with the vocabulary gather (skipped below 2 GPUs)
# ------------------------------------------------------------------------------------------------------------------

def _tp_worker(rank, ws, port, q):
    import torch
    import torch.distributed as dist
    from tests.test_tp_picks_gpu import _allgather, _device
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = _device(rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=ws)
    res = {}
    try:
        from zhilight_b200 import dist as zdist, ops
        from zhilight_b200.llama import LlamaDecoder
        V, MS = TINY["vocab_size"], 64
        sd = omodel.make_state_dict(TINY, 5, 128, False, seed=6)
        comm = zdist.TPComm(16 * TINY["dim_model"], rank, ws)
        dec = LlamaDecoder(quant_type=5, max_batch=4, max_seq=MS, tp_rank=rank, tp_size=ws, prefill_chunk=16, **TINY)
        dec.set_comm(comm)
        dec.load_state_dict(zdist.shard_state_dict(sd, rank, ws))
        dec.enable_tp_picks()
        aut, seqs = _choices(V)
        dec.enable_constraints(aut.n_states, aut.n_edges)
        params = [dict(temperature=0.0), dict(temperature=0.8, seed=4), dict(temperature=1.5, top_k=5, seed=9),
                  dict(temperature=1.0, seed=2)]

        # per-step one-state masks: the single-GPU zl_sample_masked over the concatenated shards, on every rank
        for t, p in enumerate(params):
            dec.set_sampling(t, **p)
        rng = np.random.default_rng(0)   # the same masks on every rank
        tok, ok = np.array([5, 9, 3, 12], np.int32), True
        for pos in range(8):
            masks = np.stack([C.token_bitmask(rng.choice(V, (1, 10, V // 2)[(t + pos) % 3], replace=False), V)
                              for t in range(4)])
            for t in range(4):
                dec.set_constraint(t, C.allowed(bitmask=masks[t], vocab_size=V))
            nxt, shard = dec.decode(tok, np.full(4, pos, np.int32), want_logits=True)
            full = np.concatenate(_allgather(shard), axis=1)
            want = ops.sample_masked(torch.from_numpy(full).to(dev), params, torch.from_numpy(masks.view(np.int32)).to(dev),
                                     counter=torch.full((4,), pos, dtype=torch.int32, device=dev)).cpu().numpy()
            ok = ok and np.array_equal(nxt, want) and all(np.array_equal(r, nxt) for r in _allgather(nxt))
            tok = nxt.astype(np.int32)
        res["masks"] = bool(ok)

        # a choices trie: a host loop of decode steps (states checked after each) and generate agree on every rank
        rules = [([1, 2], 0)] * 3 + [((), 6)]
        tok0, pos0 = np.array([5, 9, 3, 12], np.int32), np.array([1, 2, 3, 4], np.int32)

        def arm():
            for t in range(4):
                dec.set_sampling(t, **params[t])
                dec.set_constraint(t, aut if t < 3 else None)

        arm()
        tok, pos = tok0.copy(), pos0.copy()
        out, fin, states_ok = [[] for _ in range(4)], np.zeros(4, np.int32), True
        prev = dec.constraint_state(4)
        for _ in range(10):
            if fin.all():
                break
            live = fin == 0
            nxt = dec.decode(np.where(live, tok, 0), np.where(live, pos, MS - 1))
            st = dec.constraint_state(4)
            for t in np.nonzero(live)[0]:
                x = int(nxt[t])
                out[t].append(x)
                if t < 3:
                    states_ok = states_ok and st[t] == aut.next_state(int(prev[t]), x)
                ids, budget = rules[t]
                if x in ids:
                    fin[t] = 1
                elif budget and len(out[t]) >= budget:
                    fin[t] = 2
                tok[t], pos[t] = x, pos[t] + 1
            prev = st
        arm()
        dec.set_state(tok0, pos0)
        for t, r in enumerate(rules):
            dec.set_stop(t, *r)
        got, gfin, _ = dec.generate(4, 10)
        gstate = dec.constraint_state(4)
        mine = ([list(map(int, g)) for g in got], list(map(int, gfin)), list(map(int, gstate)))
        res["states"] = bool(states_ok)
        res["generate"] = bool(mine[0] == out and mine[1] == list(map(int, fin))
                               and all(f == 1 and o[:-1] in seqs and o[-1] in (1, 2) for f, o in zip(gfin[:3], out[:3]))
                               and all(gstate[t] == co.run_automaton(aut, out[t])[-1] for t in range(3))
                               and gstate[3] == -1 and all(o == mine for o in _allgather(mine)))
        dec.close()
        comm.close()
    except Exception:   # pragma: no cover
        import traceback
        res["error"] = traceback.format_exc()
    finally:
        q.put((rank, res))
        dist.destroy_process_group()


@pytest.mark.parametrize("ws", [2])
def test_tp_constraints(lib, cuda, ws):
    import torch
    from tests.test_tp_picks_gpu import _spawn
    if torch.cuda.device_count() < ws:
        pytest.skip("needs %d GPUs" % ws)
    results = _spawn(ws, target=_tp_worker)
    for r in range(ws):
        res = results[r]
        assert "error" not in res, res.get("error")
        assert res["masks"] and res["states"] and res["generate"], res
