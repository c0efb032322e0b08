"""Constrained decoding without a GPU: the automaton builders, the validation of TokenAutomaton and of the C-ABI
(zl_token_automaton_check, the refusals before a model is touched), and the masked pick of tests/constraint_oracle.py."""
import ctypes

import numpy as np
import pytest

from tests import constraint_oracle as co
from tests import sampling_oracle as so
from zhilight_b200 import constraints as C

INVALID = -1
V = 1000   # not a multiple of 32: the last mask word has tail bits


def _c_check(lib, a):
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    return lib.zl_token_automaton_check(a["vocab"], a["masks"].shape[0], p(a["masks"]), p(a["row_ptr"]),
                                        a["edge_tok"].size, p(a["edge_tok"]), p(a["edge_next"]), p(a["default_next"]),
                                        a["start"])


def _arrays(aut):
    return dict(vocab=aut.vocab_size, masks=aut.masks.copy(), row_ptr=aut.row_ptr.copy(), edge_tok=aut.edge_tok.copy(),
                edge_next=aut.edge_next.copy(), default_next=aut.default_next.copy(), start=aut.start)


def _automaton(a):
    return C.TokenAutomaton(a["vocab"], a["masks"], a["row_ptr"], a["edge_tok"], a["edge_next"], a["default_next"],
                            a["start"])


def test_bitmask_layout():
    m = C.token_bitmask([0, 31, 32, 999], V)
    assert m.dtype == np.uint32 and m.shape == (32,)
    assert m[0] == 0x80000001 and m[1] == 1 and m[31] == 1 << (999 - 992)
    assert list(C.bitmask_tokens(m)) == [0, 31, 32, 999]


def test_allowed_builder():
    a = C.allowed([5, 700, 3], V)
    assert a.n_states == 1 and a.n_edges == 0 and list(a.default_next) == [0] and a.start == 0
    assert list(a.allowed_tokens(0)) == [3, 5, 700]
    assert a.next_state(0, 5) == 0
    b = C.allowed(bitmask=C.token_bitmask([9, 10], V), vocab_size=V)   # a grammar engine's bitmask as it comes
    assert list(b.allowed_tokens(0)) == [9, 10]
    ids = np.arange(0, 64, 2, dtype=np.uint32)             # 32 uint32 token ids at V = 1000 stay token ids
    assert ids.size == C.mask_words(V) and list(C.allowed(ids, V).allowed_tokens(0)) == list(range(0, 64, 2))
    for kw in (dict(), dict(tokens=[1], bitmask=C.token_bitmask([1], V)), dict(bitmask=np.ones(32, np.int32)),
               dict(bitmask=np.ones(31, np.uint32))):
        with pytest.raises(ValueError):
            C.allowed(vocab_size=V, **kw)
    with pytest.raises(ValueError):
        C.allowed([1])                                      # no vocabulary size
    with pytest.raises(ValueError):
        C.allowed([], V)                                    # empty mask
    with pytest.raises(ValueError):
        C.allowed([V], V)


def test_choices_trie_with_a_prefix_choice():
    """'yes' = [7], 'yes please' = [7, 8, 9], 'no' = [4, 2]: the node after 7 allows the end ids and 8."""
    a = C.choices([[7, 8, 9], [7], [4, 2], [7]], end_ids=[1, 0], vocab_size=V)
    root = a.start
    assert list(a.allowed_tokens(root)) == [4, 7]
    s7 = a.next_state(root, 7)
    assert list(a.allowed_tokens(s7)) == [0, 1, 8]
    s78 = a.next_state(s7, 8)
    assert list(a.allowed_tokens(s78)) == [9]
    s789 = a.next_state(s78, 9)
    assert list(a.allowed_tokens(s789)) == [0, 1]
    final = a.next_state(s789, 1)
    assert a.next_state(s7, 0) == final and list(a.allowed_tokens(final)) == [0, 1]
    assert a.next_state(final, 1) == final
    s4 = a.next_state(root, 4)
    assert list(a.allowed_tokens(s4)) == [2]
    assert list(a.allowed_tokens(a.next_state(s4, 2))) == [0, 1]
    # every path from the start that follows allowed tokens spells one choice, then ends
    assert a.n_states == 7   # root, 7, 78, 789, 4, 42, final
    assert co.run_automaton(a, [7, 8, 9, 0])[-1] == final


@pytest.mark.parametrize("seqs,ends", [
    ([], [0]), ([[]], [0]), ([[1]], []),        # nothing to choose, an empty choice, no end id
    ([[1, 2]], [2]),                            # an end id inside a choice
    ([[1, V]], [0]), ([[1]], [-1]),             # ids out of range
])
def test_choices_refuses(seqs, ends):
    with pytest.raises(ValueError):
        C.choices(seqs, ends, V)


def _bad_cases():
    base = _arrays(C.choices([[7, 8, 9], [4, 2]], [1], V))
    cases = {}

    def case(name, **kw):
        a = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in base.items()}
        for k, f in kw.items():
            f(a) if callable(f) else a.__setitem__(k, f)
        cases[name] = a

    def zero_mask(a):
        a["masks"][2] = 0
    def tail_bit(a):
        a["masks"][0, -1] |= np.uint32(1 << 30)   # token 1022 >= V
    def row_start(a):
        a["row_ptr"][0] = 1
    def row_decrease(a):
        a["row_ptr"][1], a["row_ptr"][2] = a["row_ptr"][2], a["row_ptr"][1]
    def row_end(a):
        a["row_ptr"][-1] -= 1
    def unsorted(a):
        a["edge_tok"][0], a["edge_tok"][1] = a["edge_tok"][1], a["edge_tok"][0]
    def repeated(a):
        a["edge_tok"][1] = a["edge_tok"][0]
    def outside_mask(a):
        a["edge_tok"][a["row_ptr"][1]] = 5        # state 1 allows 8 only
    def edge_next(a):
        a["edge_next"][0] = a["masks"].shape[0]
    def edge_next_neg(a):
        a["edge_next"][0] = -1
    def default(a):
        a["default_next"][1] = a["masks"].shape[0]
    def edge_oob(a):
        a["edge_tok"][-1] = V
    case("empty mask", f=zero_mask)
    case("tail bit", f=tail_bit)
    case("row_ptr start", f=row_start)
    case("row_ptr decreasing", f=row_decrease)
    case("row_ptr end", f=row_end)
    case("unsorted edges", f=unsorted)
    case("repeated edge token", f=repeated)
    case("edge token outside the mask", f=outside_mask)
    case("edge token out of range", f=edge_oob)
    case("edge next out of range", f=edge_next)
    case("edge next negative", f=edge_next_neg)
    case("default out of range", f=default)
    case("start out of range", start=base["masks"].shape[0])
    case("negative start", start=-1)
    return base, cases


def test_validation_accepts_built_automata(lib):
    base, _ = _bad_cases()
    _automaton(base)
    assert _c_check(lib, base) == 0
    a = _arrays(C.allowed([0, V - 1], V))
    assert _c_check(lib, a) == 0


@pytest.mark.parametrize("name", sorted(_bad_cases()[1]))
def test_validation_refuses(lib, name):
    """TokenAutomaton and zl_token_automaton_check refuse the same malformed automata."""
    a = _bad_cases()[1][name]
    with pytest.raises(ValueError):
        _automaton(a)
    assert _c_check(lib, a) == INVALID


def test_c_check_refuses_shapes_and_nulls(lib):
    a = _arrays(C.allowed([3], V))
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    m, r, d = p(a["masks"]), p(a["row_ptr"]), p(a["default_next"])
    assert lib.zl_token_automaton_check(V, 0, m, r, 0, None, None, d, 0) == INVALID      # no state
    assert lib.zl_token_automaton_check(0, 1, m, r, 0, None, None, d, 0) == INVALID      # no vocabulary
    assert lib.zl_token_automaton_check(V, 1, None, r, 0, None, None, d, 0) == INVALID
    assert lib.zl_token_automaton_check(V, 1, m, None, 0, None, None, d, 0) == INVALID
    assert lib.zl_token_automaton_check(V, 1, m, r, 0, None, None, None, 0) == INVALID
    assert lib.zl_token_automaton_check(V, 1, m, r, 1, None, None, d, 0) == INVALID      # edges without arrays
    assert lib.zl_token_automaton_check(V, 1, m, r, -1, None, None, d, 0) == INVALID


def test_null_model_refusals(lib):
    a = _arrays(C.allowed([3], V))
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    out = np.zeros(4, np.int32)
    assert lib.zl_llama_enable_constraints(None, 4, 4) == INVALID
    assert lib.zl_llama_set_constraint(None, 0, 1, p(a["masks"]), p(a["row_ptr"]), 0, None, None,
                                       p(a["default_next"]), 0) == INVALID
    assert lib.zl_llama_get_constraint_state(None, p(out), 1) == INVALID


def test_header_declares_the_entry_points():
    from zhilight_b200 import _lib
    pr = _lib.parse_header()
    assert [a for _, a in pr["zl_sample_masked"][1]][16:19] == ["masks", "mask_words", "mask_row"]
    assert [a for _, a in pr["zl_llama_set_constraint"][1]] == [
        "m", "task", "n_states", "masks_host", "row_ptr_host", "n_edges", "edge_tok_host", "edge_next_host",
        "default_next_host", "start"]
    assert [a for _, a in pr["zl_llama_enable_constraints"][1]] == ["m", "max_states", "max_edges"]
    assert [a for _, a in pr["zl_llama_get_constraint_state"][1]] == ["m", "states_host", "B"]


def test_oracle_masked_greedy():
    l = np.array([5.0, 1.0, 3.0, 3.0, 9.0, np.nan], np.float32)
    assert co.masked_pick(l, [1, 2, 3])[0] == 2          # lowest-index maximum over the allowed tokens
    assert co.masked_pick(l, [1, 5])[0] == 1             # an allowed NaN counts as -inf
    assert co.masked_pick(l, [4])[0] == 4
    assert co.masked_pick(l, C.bitmask_tokens(C.token_bitmask([0, 3], 6)))[0] == 0


def test_oracle_all_allowed_banned_by_bias():
    l = np.array([5.0, 1.0, 3.0, 3.0, 9.0], np.float32)
    bias = {1: -np.inf, 3: -np.inf}
    for params in (None, dict(temperature=0.8, seed=3), dict(temperature=1.0, top_k=1)):
        assert co.masked_pick(l, [1, 3], params=params, bias=bias) == (1, False)
    # one allowed token left finite takes the pick
    assert co.masked_pick(l, [1, 2, 3], params=dict(temperature=0.8, seed=3), bias=bias)[0] == 2


def test_oracle_sampled_pick_stays_allowed_and_counts_top_k_over_allowed():
    rng = np.random.default_rng(0)
    l = rng.normal(size=64).astype(np.float32)
    allowed = np.sort(rng.choice(64, size=10, replace=False))
    order = allowed[np.argsort(-l[allowed], kind="stable")]
    seen = set()
    for c in range(400):
        tok, _ = co.masked_pick(l, allowed, params=dict(temperature=1.0, top_k=3, seed=11), counter=c)
        seen.add(tok)
    assert seen <= set(order[:3].tolist()) and len(seen) == 3   # the top 3 of the allowed tokens, all drawn
    # the masked pick is the plain pick of the row with the masked tokens at -inf (same u)
    lm = np.full_like(l, -np.inf)
    lm[allowed] = l[allowed]
    for c in range(50):
        u = float(so.uniform(11, c))
        want, _ = so.pick(lm, 0.7, 0.9, 0, u)
        assert co.masked_pick(l, allowed, params=dict(temperature=0.7, top_p=0.9, seed=11), counter=c)[0] == want
