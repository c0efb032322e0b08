"""zl_sample on the GPU against the numpy contract (tests/sampling_oracle.py), and the decode driver's sampled steps."""
import numpy as np
import pytest
from scipy import stats

from oracle import model as omodel
from tests import sampling_oracle as so
from tests.test_llama_gpu import TINY

pytestmark = pytest.mark.gpu


def _t(a, dev, dtype=None):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev) if dtype is None else torch.tensor(a, dtype=dtype, device=dev)


def _sample(dev, logits, params, row_task=None, counter=None, history=None):
    """-> (tokens, history after) as numpy"""
    import torch
    from zhilight_b200 import ops
    rt = None if row_task is None else _t(np.asarray(row_task, dtype=np.int32), dev)
    ct = None if counter is None else _t(np.asarray(counter, dtype=np.int32), dev)
    h = None if history is None else _t(np.asarray(history, dtype=np.int32), dev)
    out = ops.sample(_t(np.asarray(logits, dtype=np.float32), dev), params, rt, ct, h)
    torch.cuda.synchronize()
    return out.cpu().numpy(), (None if h is None else h.cpu().numpy())


def _random_params(rng, greedy_share=0.15):
    if rng.random() < greedy_share:
        return dict(temperature=0.0, seed=int(rng.integers(0, 2 ** 63)))
    return dict(temperature=float(rng.choice([0.3, 0.7, 1.0, 1.5])), top_p=float(rng.choice([1.0, 1.0, 0.95, 0.6])),
                top_k=int(rng.choice([0, 0, 5, 50, 2000])),
                repetition_penalty=float(rng.choice([1.0, 1.3, 0.8])), presence_penalty=float(rng.choice([0.0, 0.0, 0.7])),
                seed=int(rng.integers(0, 2 ** 64, dtype=np.uint64)))


def _rows(rng, n, V, kind):
    if kind == "normal":
        return (rng.normal(size=(n, V)) * 3).astype(np.float32)
    if kind == "ties":
        l = (np.round(rng.normal(size=(n, V)) * 2) / 2).astype(np.float32)
        l[:, ::7] = -np.inf
        return l
    if kind in ("lm", "lm_ties"):
        # language-model-like rows: a few dozen head tokens carry most of the mass above a wide flat tail (with a
        # flat 128K-token tail most targets would land among tokens lighter than the 1e-5 ambiguity margin)
        l = (rng.normal(size=(n, V)) * 2).astype(np.float32)
        for r in range(n):
            head = rng.choice(V, size=64, replace=False)
            l[r, head] += rng.uniform(14, 24, size=64).astype(np.float32)
        if kind == "lm_ties":
            l = np.round(l * 2) / 2
            l[:, ::7] = -np.inf
        return l.astype(np.float32)
    raise ValueError(kind)


@pytest.mark.parametrize("V,n,kinds", [(1000, 400, ("normal", "ties")), (128256, 128, ("lm", "lm_ties"))])
def test_exact_picks_match_oracle(lib, cuda, V, n, kinds):
    rng = np.random.default_rng(V)
    logits = np.concatenate([_rows(rng, n // 2, V, kinds[0]), _rows(rng, n - n // 2, V, kinds[1])])
    params = [_random_params(rng) for _ in range(n)]
    counter = rng.integers(0, 2 ** 31, size=n).astype(np.int32)
    hist_tokens = [set(rng.integers(0, V, size=int(rng.integers(0, 40))).tolist()) for _ in range(n)]
    history = so.history_bitmap(hist_tokens, V)
    got, h_after = _sample(cuda, logits, params, None, counter, history)
    amb = 0
    for i in range(n):
        p = params[i]
        pen = so.penalise(logits[i], hist_tokens[i], p.get("repetition_penalty", 1.0), p.get("presence_penalty", 0.0))
        u = float(so.uniform(p["seed"], int(counter[i])))
        want, ambiguous = so.pick(pen, p["temperature"], p.get("top_p", 1.0), p.get("top_k", 0), u)
        assert 0 <= got[i] < V
        if ambiguous:
            amb += 1
            continue
        assert got[i] == want, (i, p, got[i], want)
        # the pick is recorded in the task's history, nothing else changes
        assert so.bitmap_tokens(h_after[i], V) == hist_tokens[i] | {int(got[i])}
    assert amb < 0.01 * n


def _chi2_check(draws, p):
    V = p.size
    counts = np.bincount(draws, minlength=V)
    assert counts[p == 0].sum() == 0, "draw outside the oracle's support"
    exp = p * draws.size
    big = exp >= 5
    obs_m = np.concatenate([counts[big], [counts[~big].sum()]])
    exp_m = np.concatenate([exp[big], [exp[~big].sum()]])
    if exp_m[-1] == 0:
        obs_m, exp_m = obs_m[:-1], exp_m[:-1]
    exp_m = exp_m * obs_m.sum() / exp_m.sum()
    return stats.chisquare(obs_m, exp_m).pvalue


DIST = {
    "temperature": dict(temperature=0.8),
    "top_k": dict(temperature=1.0, top_k=20),
    "top_p": dict(temperature=0.9, top_p=0.8),
    "top_k_top_p": dict(temperature=1.1, top_k=30, top_p=0.9),
    "penalties": dict(temperature=1.0, repetition_penalty=1.5),
    "presence": dict(temperature=1.0, top_p=0.95, presence_penalty=1.0),
    "ties": dict(temperature=1.0, top_k=12),
}


@pytest.mark.parametrize("name", list(DIST))
def test_distribution_matches_oracle(lib, cuda, name):
    """65536 draws in one launch: the rows share logits and parameters and differ by their counter."""
    N, V = 65536, 256
    rng = np.random.default_rng(list(DIST).index(name))
    row = _rows(rng, 1, V, "ties" if name == "ties" else "normal")[0] * (0.5 if name != "ties" else 1.0)
    p = dict(DIST[name], seed=1234)
    hist_tokens = set(np.argsort(-row)[:6].tolist()) if "penalty" in str(p) else set()
    logits = np.broadcast_to(row, (N, V))
    if hist_tokens:
        # one task per row with the same history (a history must not be shared between rows)
        history = np.broadcast_to(so.history_bitmap([hist_tokens], V), (N, (V + 31) // 32))
        draws, _ = _sample(cuda, logits, [p] * N, None, np.arange(N), history)
    else:
        draws, _ = _sample(cuda, logits, [p], np.zeros(N), np.arange(N))
    pen = so.penalise(row, hist_tokens, p.get("repetition_penalty", 1.0), p.get("presence_penalty", 0.0))
    probs = so.probs(pen, p["temperature"], p.get("top_p", 1.0), p.get("top_k", 0))
    assert _chi2_check(draws, probs) >= 1e-4


@pytest.mark.parametrize("V", [1000, 128256])
def test_greedy_rows_equal_argmax(lib, cuda, V):
    import torch
    from zhilight_b200 import ops
    rng = np.random.default_rng(7)
    n = 24
    logits = np.concatenate([_rows(rng, n // 2, V, "normal"), _rows(rng, n // 2, V, "ties")])
    logits[3, 10] = logits[3, 500] = logits[3].max() + 1   # an exact tie on the maximum
    params = []
    for i in range(n):
        if i % 3 == 0:
            params.append(dict(temperature=0.0))
        elif i % 3 == 1:
            params.append(dict(temperature=0.8, top_k=1, top_p=0.5, seed=i))
        else:
            params.append(dict(temperature=0.8, top_p=0.9, seed=i))
    got, _ = _sample(cuda, logits, params, None, np.arange(n))
    ref = ops.argmax(_t(logits, cuda)).cpu().numpy()
    torch.cuda.synchronize()
    greedy_rows = [i for i in range(n) if i % 3 != 2]
    np.testing.assert_array_equal(got[greedy_rows], ref[greedy_rows])
    assert got[3] == 10


def test_reproducible_and_permutation_equivariant(lib, cuda):
    rng = np.random.default_rng(3)
    n, V = 64, 5000
    logits = _rows(rng, n, V, "normal")
    params = [_random_params(rng, 0.2) for _ in range(n)]
    counter = rng.integers(0, 1000, size=n)
    hist = so.history_bitmap([set(rng.integers(0, V, 10).tolist()) for _ in range(n)], V)
    a, ha = _sample(cuda, logits, params, None, counter, hist)
    b, hb = _sample(cuda, logits, params, None, counter, hist)
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(ha, hb)
    perm = rng.permutation(n)
    c, hc = _sample(cuda, logits[perm], params, perm, counter[perm], hist)   # row i is task perm[i]
    np.testing.assert_array_equal(c, a[perm])
    np.testing.assert_array_equal(hc, ha)


def test_degenerate_rows_stay_in_range(lib, cuda):
    V = 3000
    logits = np.zeros((4, V), dtype=np.float32)
    logits[0] = -np.inf                     # nothing finite: greedy fallback (index 0)
    logits[1, :] = -np.inf
    logits[1, 1234] = 0.0                   # one finite token
    logits[2, 77] = np.inf                  # +inf maximum: greedy fallback
    logits[3, ::2] = np.nan                 # NaN has probability 0
    got, _ = _sample(cuda, logits, dict(temperature=1.0, seed=9), None, np.arange(4))
    assert got[0] == 0 and got[1] == 1234 and got[2] == 77
    assert got[3] % 2 == 1


# ------------------------------------------------------------------------------------------ decode driver
SAMPLED = {1: dict(temperature=0.9, top_p=0.9, top_k=50, repetition_penalty=1.3, seed=11),
           2: dict(temperature=1.2, presence_penalty=0.5, seed=5)}


def _drive(cuda, sd, quant, graph, mode, steps=6):
    """Task 0 greedy, tasks 1 and 2 sampled.  Every pick must equal ops.sample on the step's own logits with the same
    history / counter; task 1 is prefilled first and its sampling is set again (history cleared) mid-way."""
    from zhilight_b200.llama import LlamaDecoder
    V = TINY["vocab_size"]
    dec = LlamaDecoder(quant_type=quant, dtype="f16", max_batch=3, max_seq=64, use_graph=graph, prefill_chunk=16, **TINY)
    dec.load_state_dict(sd)
    for t, p in SAMPLED.items():
        dec.set_sampling(t, **p)
    params = [dict(temperature=0.0)] + [SAMPLED[1], SAMPLED[2]]
    hist = np.zeros((3, (V + 31) // 32), dtype=np.int32)
    # prefill task 1: the returned token is ops.sample of the returned logits at counter pos0 + n - 1
    prompt = np.arange(3, 13, dtype=np.int32)
    t1, l1 = dec.prefill(1, prompt, want_logits=True)
    want, h1 = _sample(cuda, l1, params, [1], [len(prompt) - 1], hist)
    assert t1 == want[0]
    hist = h1
    assert so.bitmap_tokens(hist[1], V) == {t1}
    tok = np.array([5, t1, 9], dtype=np.int32)
    pos = np.array([0, len(prompt), 0], dtype=np.int32)
    seq = []
    if mode == "device":
        dec.set_state(tok, pos)
    for s in range(steps):
        if s == 3:
            dec.set_sampling(1, **SAMPLED[1])
            hist[1] = 0
        if mode == "host":
            nxt = dec.decode(tok, pos)
        else:
            dec.step_device(3)
            nxt, npos = dec.get_state(3)
            np.testing.assert_array_equal(npos, pos + 1)
        logits = dec.get_logits(3)
        want, hist = _sample(cuda, logits, params, None, pos, hist)
        np.testing.assert_array_equal(nxt, want)
        assert nxt[0] == int(np.argmax(logits[0]))
        seq.append(nxt.copy())
        tok, pos = nxt, pos + 1
    dec.close()
    return np.array(seq)


@pytest.mark.parametrize("quant", [5, 0, 2], ids=["gptq", "dense", "w8a8"])
def test_driver_sampled_steps_match_ops_sample(lib, cuda, quant):
    sd = omodel.make_state_dict(TINY, quant, 128, False, seed=1, dtype="f16")
    runs = [_drive(cuda, sd, quant, graph, mode) for graph, mode in ((True, "host"), (False, "host"), (True, "device"))]
    np.testing.assert_array_equal(runs[0], runs[1])
    np.testing.assert_array_equal(runs[0], runs[2])


def test_kernels_per_step_unchanged_without_sampling(lib, cuda):
    from zhilight_b200.llama import LlamaDecoder
    sd = omodel.make_state_dict(TINY, 5, 128, False, seed=2)
    counts = []
    for setup in ("none", "greedy", "sampled"):
        dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, **TINY)
        dec.load_state_dict(sd)
        if setup == "greedy":
            dec.set_sampling(1, temperature=0.0)
        elif setup == "sampled":
            dec.set_sampling(1, temperature=0.7, seed=3)
        dec.decode(np.array([1, 2], np.int32), np.array([0, 0], np.int32))
        counts.append(dec.stats(2)[1])
        dec.close()
    assert counts[0] == counts[1]
    assert counts[2] == counts[0] - 1   # one sampler launch instead of the two argmax kernels


def test_tp_sampling_is_unsupported(lib, cuda):
    from zhilight_b200 import _lib
    from zhilight_b200.llama import LlamaDecoder
    dec = LlamaDecoder(quant_type=5, max_batch=2, max_seq=32, tp_rank=0, tp_size=2, **TINY)
    with pytest.raises(_lib.ZLError) as e:
        dec.set_sampling(0, temperature=0.8)
    assert e.value.code == -2
    dec.close()
