"""GPU checks of beam search: zl_beam_topk against a float64 top-K (dead NaN rows, exact duplicates, huge and -inf
logits, every width and K), zl_llama_kv_copy_rows bit for bit, and beam_search end to end on the decode driver -- width 1
is the greedy decode loop, the recorded candidates replay through the oracle policy to the same beams and results, each
result's cum_logprob is what teacher-forcing its tokens gives, and the step's graph keeps the decode step's launch count."""
import numpy as np
import pytest

from oracle import model as omodel
from tests import beam_oracle
from tests.test_llama_gpu import LAYER8B, TINY

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED, STATE = -1, -2, -4


def _ref_topk(logits, cum, groups, k):
    """float64 scores of every (row, token) of each group, sorted by (score desc, flat index asc)"""
    out = []
    for row0, width in groups:
        s, key = [], []
        for j in range(width):
            r = row0 + j
            if not cum[r] > -np.inf:
                continue
            x = logits[r].astype(np.float64)
            m = x.max()
            lse = m + np.log(1e-20 + np.exp(x - m).sum())
            sc = cum[r] + x - lse
            ok = np.isfinite(sc)
            s.append(sc[ok])
            key.append(j * logits.shape[1] + np.nonzero(ok)[0])
        s = np.concatenate(s) if s else np.zeros(0)
        key = np.concatenate(key) if key else np.zeros(0, np.int64)
        order = np.lexsort((key, -s))
        out.append((s[order], key[order]))
    return out


def _check_topk(logits, cum, groups, k, cuda):
    import torch
    from zhilight_b200 import ops
    parent, token, score = ops.beam_topk(torch.from_numpy(logits).to(cuda), torch.from_numpy(cum).to(cuda), groups, k)
    parent, token, score = parent.cpu().numpy(), token.cpu().numpy(), score.cpu().numpy()
    V = logits.shape[1]
    for g, (s_ref, key_ref) in enumerate(_ref_topk(logits, cum, groups, k)):
        n = min(k, s_ref.size)
        assert (parent[g, n:] == -1).all() and (token[g, n:] == -1).all() and np.isneginf(score[g, n:]).all()
        got = score[g, :n].astype(np.float64)
        tol = 2e-6 * np.maximum(1.0, np.abs(s_ref[:n])) + 1e-5
        assert np.all(np.abs(got - s_ref[:n]) <= tol), g
        key = parent[g, :n].astype(np.int64) * V + token[g, :n]
        # each returned (row, token) carries its own float64 score, and the order is exact where the gap exceeds tol
        r0 = groups[g][0]
        own = np.array([cum[r0 + p] + logits[r0 + p, v].astype(np.float64) -
                        (logits[r0 + p].astype(np.float64).max() +
                         np.log(1e-20 + np.exp(logits[r0 + p].astype(np.float64) -
                                               logits[r0 + p].astype(np.float64).max()).sum()))
                        for p, v in zip(parent[g, :n], token[g, :n])])
        assert np.all(np.abs(own - s_ref[:n]) <= 2 * tol), g
        clear = np.ones(n, bool)
        gaps = np.abs(np.diff(s_ref[:min(n + 1, s_ref.size)]))
        for i in range(n):
            if (i > 0 and gaps[i - 1] <= 2 * tol[i]) or (i < gaps.size and gaps[i] <= 2 * tol[i]):
                clear[i] = False
        assert np.array_equal(key[clear], key_ref[:n][clear]), g
        # exact duplicates: equal scores come in ascending flat index
        for i in range(n - 1):
            if got[i] == got[i + 1]:
                assert key[i] < key[i + 1]


@pytest.mark.parametrize("V", [512, 32000, 128256, 152064])
@pytest.mark.parametrize("W", [1, 2, 4, 8, 16])
def test_beam_topk_matches_float64(lib, cuda, W, V):
    rng = np.random.default_rng(W * 1000 + V % 997)
    G = 3
    R = G * W
    logits = (rng.standard_normal((R, V)) * 3).astype(np.float32)
    cum = (-rng.random(R) * 5).astype(np.float32)
    groups = [(g * W, W) for g in range(G)]
    # group 0: the first step -- one live row, the others dead and NaN-filled
    if W > 1:
        cum[1:W] = -np.inf
        logits[1:W] = np.nan
    # group 1: exact duplicates across and inside rows, a huge logit, -inf logits
    r = W
    logits[r, 5:40] = logits[r].max() + 1.0
    logits[r + W - 1, 7] = logits[r].max() + 1.0
    cum[r + W - 1] = cum[r]
    logits[r, 100:200] = -np.inf
    # group 2: huge logits and a row of -inf but one
    r = 2 * W
    logits[r, 3] = 3e4
    logits[r, 4] = 3e4
    if W > 1:
        logits[r + 1, :] = -np.inf
        logits[r + 1, 9] = 0.0
    for k in sorted({1, min(2 * W, 32), 32}):
        _check_topk(logits, cum, groups, k, cuda)


def test_beam_topk_fewer_candidates_than_k_and_refusals(lib, cuda):
    import torch
    from zhilight_b200 import _lib, ops
    logits = np.full((2, 512), -np.inf, np.float32)
    logits[0, [3, 9, 11]] = [1.0, 2.0, 1.0]
    cum = np.array([0.0, -np.inf], np.float32)
    _check_topk(logits, cum, [(0, 2)], 8, cuda)
    lt, ct = torch.from_numpy(logits).to(cuda), torch.from_numpy(cum).to(cuda)
    for groups, k, code in (([(0, 1)], 4, INVALID), ([(0, 2)], 33, INVALID), ([(0, 2)], 0, INVALID),
                            ([(1, 1), (0, 1)], 4, INVALID), ([(0, 1), (2, 1)], 4, INVALID)):
        with pytest.raises(_lib.ZLError) as e:
            ops.beam_topk(lt, ct, groups, k)
        assert e.value.code == code


def _decoder(quant=5, dtype="f16", kv=None, cfg=TINY, max_batch=8, max_seq=96, chunk=16, seed=0, **kw):
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=quant, dtype=dtype, max_batch=max_batch, max_seq=max_seq, prefill_chunk=chunk,
                       kv_cache_dtype=kv, **cfg, **kw)
    dec.load_state_dict(omodel.make_state_dict(cfg, quant, 128, False, seed=seed, dtype=dtype))
    return dec


COPY_KINDS = {"gptq-f16": dict(quant=5), "gptq-int8kv": dict(quant=5, kv="int8"), "bf16-dense": dict(quant=0, dtype="bf16")}


@pytest.mark.parametrize("kind", list(COPY_KINDS))
def test_kv_copy_rows_is_bit_exact_and_touches_nothing_else(lib, cuda, kind):
    from zhilight_b200 import _lib
    L, S = TINY["num_layers"], 96
    dec = _decoder(max_batch=6, max_seq=S, **COPY_KINDS[kind])
    rng = np.random.default_rng(1)
    for task in range(6):   # distinct rows in every task
        dec.prefill(task, rng.integers(0, TINY["vocab_size"], S).astype(np.int32))
    before = [[dec.read_kv(l, t, 0, S) for t in range(6)] for l in range(L)]
    ranges = np.array([[0, 1, 0, 5], [0, 2, 40, S], [3, 4, 17, 18], [3, 5, 0, S]], np.int32)
    dec.kv_copy_rows(ranges)
    for l in range(L):
        after = [dec.read_kv(l, t, 0, S) for t in range(6)]
        for t in range(6):
            want = [a.copy() for a in before[l][t]]
            for src, dst, r0, r1 in ranges:
                if dst == t:
                    for w, b in zip(want, before[l][src]):
                        w[r0:r1] = b[r0:r1]
            for w, a in zip(want, after[t]):
                assert np.array_equal(w.view(np.uint8), a.view(np.uint8)), (l, t)
    for bad in ([[0, 1, 0, 5], [2, 1, 0, 5]],      # a destination twice
                [[0, 1, 0, 5], [1, 2, 0, 5]],      # task 1 both destination and source
                [[0, 1, 0, S + 1]], [[0, 1, -1, 3]], [[0, 1, 3, 3]], [[0, 0, 0, 3]], [[0, 6, 0, 3]]):
        with pytest.raises(_lib.ZLError) as e:
            dec.kv_copy_rows(np.array(bad, np.int32))
        assert e.value.code == INVALID
    dec.close()


def _rescore(dec, prompt, tokens, eos, max_new, batch):
    """cum log-probability of prompt -> tokens (+ EOS when the result ended early) teacher-forced in task 0, stepped at
    the beam step's batch size so that the same GEMM routes run"""
    ended_by_eos = len(tokens) < max_new
    seq = list(prompt) + list(tokens) + ([eos] if ended_by_eos else [])
    if len(prompt) > 1:
        dec.prefill(0, np.array(prompt[:-1], np.int32))
    total = 0.0
    for i in range(len(prompt) - 1, len(seq) - 1):
        tok = np.zeros(batch, np.int32)
        pos = np.zeros(batch, np.int32)
        tok[0], pos[0] = seq[i], i
        _, logits = dec.decode(tok, pos, want_logits=True)
        x = logits[0].astype(np.float64)
        m = x.max()
        total += x[seq[i + 1]] - m - np.log(1e-20 + np.exp(x - m).sum())
    return total, len(seq) - len(prompt)


E2E = {
    "tiny-gptq": dict(cfg=TINY, quant=5),
    "tiny-gptq-int8kv": dict(cfg=TINY, quant=5, kv="int8"),
    "tiny-dense": dict(cfg=TINY, quant=0),
    "tiny-dense-int8kv": dict(cfg=TINY, quant=0, kv="int8"),
    "8b-gptq": dict(cfg=LAYER8B, quant=5),
    "8b-gptq-int8kv": dict(cfg=LAYER8B, quant=5, kv="int8"),
    "8b-dense": dict(cfg=LAYER8B, quant=0),
}


@pytest.mark.parametrize("kind", list(E2E))
def test_beam_search_end_to_end(lib, cuda, kind):
    kw = dict(E2E[kind])
    cfg = kw.pop("cfg")
    V = cfg["vocab_size"]
    W, NEW, NRES = 4, 12, 2
    dec = _decoder(cfg=cfg, max_batch=2 * W, max_seq=64, **kw)
    rng = np.random.default_rng(7)
    prompts = [list(rng.integers(0, V, 9)), list(rng.integers(0, V, 1))]
    # width 1 is the greedy decode loop
    greedy = []
    for p in prompts:
        nxt = dec.prefill(0, np.array(p, np.int32)) if len(p) > 1 else int(dec.decode([p[0]], [0])[0])
        toks = [nxt]
        for i in range(NEW - 1):
            toks.append(int(dec.decode([toks[-1]], [len(p) + i])[0]))
        greedy.append(toks)
    w1 = dec.beam_search(prompts, 1, NEW, eos_id=-1)
    assert [r[0][0] for r in w1] == greedy
    # an EOS that the search meets: the greedy run's 6th token of prompt 0
    eos = greedy[0][5]
    trace = []
    res = dec.beam_search(prompts, W, NEW, eos_id=eos, num_results=NRES, trace=trace)
    want, beams = beam_oracle.replay(trace, prompts, W, NEW, eos, NRES)
    assert res == want
    assert [rec["beams"] for rec in trace] == beams
    assert all(1 <= len(r) <= NRES for r in res)
    # every result's cum_logprob is its teacher-forced log-probability, and its score that over its length
    diffs = []
    for p, rs in zip(prompts, res):
        for tokens, score, cum in rs:
            tf, n = _rescore(dec, p, tokens, eos, NEW, 2 * W)
            diffs.append(abs(tf - cum))
            assert abs(score - cum / n) <= 1e-6 * max(1.0, abs(score))
    print("%s: |teacher-forced - reported cum_logprob| max %.3g over %d results" % (kind, max(diffs), len(diffs)))
    # measured on an H100: at most 4.5e-6 over the seven kinds (the same GEMM routes run; lse is summed in another order)
    assert max(diffs) <= 1e-4
    dec.close()


def test_beam_step_graph_launches_and_refusals(lib, cuda):
    from zhilight_b200 import _lib
    dec = _decoder(max_batch=8)
    B = 8
    tok = np.arange(B, dtype=np.int32)
    pos = np.zeros(B, np.int32)
    dec.decode(tok, pos)
    decode_launches = dec.stats()[1]
    groups = np.array([[0, 4], [4, 4]], np.int32)
    cum = np.zeros(B, np.float32)
    dec.beam_step(tok, pos, groups, cum, 8)
    # zl_argmax's two launches give way to zl_beam_topk's two
    assert dec.stats()[1] == decode_launches
    for g, c, k, code in (([[0, 4], [4, 3]], cum, 8, INVALID), ([[0, 4], [4, 4], [8, 1]], cum, 8, INVALID),
                          (groups, cum, 33, INVALID), (groups, np.full(B, np.nan, np.float32), 8, INVALID)):
        with pytest.raises(_lib.ZLError) as e:
            dec.beam_step(tok, pos, np.array(g, np.int32), c, k)
        assert e.value.code == code
    dec.set_sampling(3, temperature=0.7)
    with pytest.raises(_lib.ZLError) as e:
        dec.beam_step(tok, pos, groups, cum, 8)
    assert e.value.code == STATE
    dec.set_sampling(3)
    p1, t1, s1 = dec.beam_step(tok, pos, groups, cum, 8)
    p2, t2, s2 = dec.beam_step(tok, pos, groups, cum, 8)
    assert np.array_equal(t1, t2) and np.array_equal(s1, s2)
    dec.close()


def test_beam_step_refuses_tensor_parallelism(lib, cuda):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, tp_size=2, tp_rank=0, **TINY)
    with pytest.raises(_lib.ZLError) as e:
        dec.beam_step([1, 2], [0, 0], [[0, 2]], [0.0, -np.inf], 4)
    assert e.value.code == UNSUPPORTED
    dec.close()
