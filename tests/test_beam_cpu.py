"""CPU checks of beam search: the host policy and slot planner (zhilight_b200/beam_search.py) driven by a toy model whose
logits depend on the simulated KV rows of each slot, against the oracle (tests/beam_oracle.py); the planner's copies on
random parent maps; and the new C-ABI entry points refusing bad arguments without a GPU."""
import ctypes
import zlib

import numpy as np
import pytest

from tests import beam_oracle
from zhilight_b200 import _lib
from zhilight_b200 import beam_search as bs

INVALID, UNSUPPORTED = -1, -2
V = 50


def toy_logits(tokens, seed=0, eos=None, eos_bias=0.0):
    """reproducible logits of the next token after `tokens`"""
    h = zlib.crc32(np.asarray(tokens, np.int64).tobytes()) ^ seed
    x = np.random.default_rng(h).standard_normal(V).astype(np.float32) * 2
    if eos is not None:
        x[eos] += np.float32(eos_bias)
    return x


class ToyDriver:
    """beam_search's three entry points over simulated KV slots: a slot's rows are the tokens stepped or copied into
    them, and the logits of a step are toy_logits of the slot's rows before the position plus the input token"""

    def __init__(self, slots, max_seq, **kw):
        self.rows = np.full((slots, max_seq), -1, np.int64)
        self.kw = kw
        self.steps = 0

    def prefill(self, slot, tokens):
        self.rows[slot, :len(tokens)] = tokens

    def copy_rows(self, ranges):
        srcs = {int(r[0]) for r in ranges}
        dsts = [int(r[1]) for r in ranges]
        assert len(set(dsts)) == len(dsts) and not srcs & set(dsts)
        for s, d, r0, r1 in ranges:
            self.rows[d, r0:r1] = self.rows[s, r0:r1]

    def step(self, tokens, positions, groups, cum, k):
        self.steps += 1
        rows = []
        for s, (t, p) in enumerate(zip(tokens, positions)):
            self.rows[s, p] = t
            rows.append(beam_oracle.log_softmax_f32(toy_logits(list(self.rows[s, :p + 1]), **self.kw)))
        G = len(groups)
        parent = np.full((G, k), -1, np.int32)
        token = np.full((G, k), -1, np.int32)
        score = np.full((G, k), -np.inf, np.float32)
        for g, (r0, w) in enumerate(groups):
            for i, (p, v, sc) in enumerate(beam_oracle.topk(rows[r0:r0 + w], cum[r0:r0 + w], k)):
                parent[g, i], token[g, i], score[g, i] = p, v, sc
        return parent, token, score


def run(prompts, width, max_new, eos, num_results, seed=0, eos_bias=0.0, trace=None):
    drv = ToyDriver(len(prompts) * width, 64, seed=seed, eos=eos, eos_bias=eos_bias)
    res = bs.beam_search(drv.step, drv.copy_rows, drv.prefill, prompts, width, max_new, eos, num_results, trace)
    want = beam_oracle.search(lambda toks: toy_logits(toks, seed, eos, eos_bias), prompts, width, max_new, eos,
                              num_results)
    return res, want, drv


PROMPTS = [[3, 1, 4, 1, 5], [9], [2, 6]]


@pytest.mark.parametrize("width", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_policy_matches_oracle(width, seed):
    res, want, _ = run(PROMPTS, width, 7, eos=-1, num_results=2, seed=seed)
    assert res == want
    assert all(len(r) == 2 for r in res)


def test_width_1_is_the_greedy_loop():
    res, want, _ = run(PROMPTS, 1, 9, eos=-1, num_results=1)
    assert res == want
    for p, r in zip(PROMPTS, res):
        toks = list(p)
        for _ in range(9):
            toks.append(int(np.argmax(toy_logits(toks))))
        assert r[0][0] == toks[len(p):]


@pytest.mark.parametrize("bias", [1.0, 2.5, 4.0, 8.0])
@pytest.mark.parametrize("width", [2, 4])
def test_eos_inside_and_beyond_the_first_candidates(width, bias):
    """an EOS bias from rare to dominant: EOS among the first W candidates, after them, and ending every group early"""
    for seed in range(4):
        res, want, drv = run(PROMPTS, width, 8, eos=7, num_results=3, seed=seed, eos_bias=bias)
        assert res == want
        for r in res:
            assert all(7 not in toks for toks, _, _ in r)


def test_early_stop_and_more_results_than_beams():
    # a dominant EOS fills the results at once: the groups stop long before max_new_tokens
    trace = []
    res, want, drv = run(PROMPTS, 2, 30, eos=7, num_results=5, eos_bias=9.0, trace=trace)
    assert res == want and len(trace) < 30
    assert max(len(r) for r in res) > 2     # num_results > W
    for r in res:
        assert [s for _, s, _ in r] == sorted((s for _, s, _ in r), reverse=True)


def test_max_new_tokens_ends_every_beam():
    res, want, _ = run(PROMPTS, 4, 3, eos=-1, num_results=6)
    assert res == want
    assert all(len(toks) == 3 for r in res for toks, _, _ in r)
    for r in res:
        for toks, score, cum in r:
            assert np.float32(score) == np.float32(cum) / np.float32(3)


@pytest.mark.parametrize("seed", range(40))
def test_planner_copies_rebuild_every_slot(seed):
    rng = np.random.default_rng(seed)
    W = int(rng.integers(1, 17))
    L = int(rng.integers(1, 12))
    # slot histories: a common prompt, then random divergence; some slots shorter (dead earlier)
    base = list(rng.integers(0, 5, L))
    kv = []
    for j in range(W):
        h = list(base)
        cut = int(rng.integers(0, L + 1))
        h[cut:] = [int(x) for x in rng.integers(0, 3, L - cut)]
        if rng.random() < 0.2:
            h = h[:int(rng.integers(0, L + 1))]
        kv.append(h)
    full = [j for j in range(W) if len(kv[j]) == L]
    if not full:
        kv[0] = list(base)
        full = [0]
    n_children = int(rng.integers(1, W + 1))
    parents = [int(rng.choice(full)) for _ in range(n_children)]
    slots, copies = bs.plan_slots(parents, kv)
    assert len(set(slots)) == len(slots)
    srcs, dsts = {c[0] for c in copies}, [c[1] for c in copies]
    assert not srcs & set(dsts) and len(set(dsts)) == len(dsts)
    sim = [list(h) + [-1] * (L + 1 - len(h)) for h in kv]
    for s, d, r0, r1 in copies:
        assert 0 <= r0 < r1 <= L
        sim[d][r0:r1] = sim[s][r0:r1]
    for p, d in zip(parents, slots):
        assert sim[d][:L] == kv[p][:L]
    # a parent's first child stays in its slot
    for p in set(parents):
        assert slots[parents.index(p)] == p


def test_result_manager_replaces_the_first_minimum():
    for cls in (bs.BeamResults, None):
        m = bs.BeamResults(2) if cls else beam_oracle.ResultManager(2)
        add = m.add_result if cls else (lambda t, c, s: m.add(t, c, s))
        acc = m.accept_score if cls else m.accept
        add([1], np.float32(-1), np.float32(-1))
        add([2], np.float32(-2), np.float32(-2))
        assert acc(np.float32(-2)) and not acc(np.float32(-2.5))
        add([3], np.float32(-2), np.float32(-2))      # equal to the minimum: accepted, replaces nothing
        add([4], np.float32(-1.5), np.float32(-1.5))
        assert [t for t, _, _ in m.best()] == [[1], [4]]


def test_search_refuses_bad_widths():
    drv = ToyDriver(4, 16)
    for w in (0, 17):
        with pytest.raises(ValueError):
            bs.beam_search(drv.step, drv.copy_rows, drv.prefill, [[1]], w, 4, 0)
    with pytest.raises(ValueError):
        bs.beam_search(drv.step, drv.copy_rows, drv.prefill, [[]], 2, 4, 0)


def test_header_exports_the_beam_entry_points(lib):
    protos = _lib.parse_header()
    for name in ("zl_beam_topk", "zl_beam_topk_workspace_bytes", "zl_llama_beam_step", "zl_llama_kv_copy_rows"):
        assert name in protos, name
        assert hasattr(lib, name), name


def test_entry_points_refuse_bad_arguments_without_a_gpu(lib):
    buf = np.zeros(1 << 16, np.float32)   # stands in for device memory: nothing may touch it
    p = buf.ctypes.data_as(ctypes.c_void_p)

    def topk(R, V, groups, K, ws_bytes=1 << 30):
        g = np.ascontiguousarray(groups, np.int32).reshape(-1, 2)
        return lib.zl_beam_topk(p, R, V, p, g.ctypes.data_as(ctypes.c_void_p), g.shape[0], K, p, p, p, p, ws_bytes, 0,
                                None)

    assert topk(8, 1000, [[0, 4], [4, 4]], 0) == INVALID
    assert topk(8, 1000, [[0, 4], [4, 4]], 33) == INVALID
    assert topk(8, 1000, [[0, 4], [5, 3]], 4) == INVALID        # a gap
    assert topk(8, 1000, [[0, 4], [4, 3]], 4) == INVALID        # does not reach R
    assert topk(8, 1000, [[0, 4], [4, 5]], 4) == INVALID        # past R
    assert topk(17, 1000, [[0, 17]], 4) == INVALID              # width > 16
    assert topk(2, 1000, [[0, 0], [0, 2]], 4) == INVALID        # empty group
    assert topk(2, 262145, [[0, 2]], 4) == UNSUPPORTED
    assert topk(2, 1000, [[0, 2]], 4, ws_bytes=16) == INVALID
    assert lib.zl_beam_topk(None, 2, 1000, p, p, 1, 4, p, p, p, p, 1 << 30, 0, None) == INVALID
    assert b"invalid argument" in lib.zl_last_error()
    assert lib.zl_beam_topk_workspace_bytes(0, 1000, 4) == 0
    assert lib.zl_beam_topk_workspace_bytes(4, 128256, 32) > 0
    ranges = np.array([[0, 1, 0, 4]], np.int32)
    assert lib.zl_llama_kv_copy_rows(None, ranges.ctypes.data_as(ctypes.c_void_p), 1) == INVALID
    assert lib.zl_llama_beam_step(None, p, p, 2, p, 1, p, 4, p, p, p, None) == INVALID
