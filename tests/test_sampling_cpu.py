"""Sampling contract without a GPU: the Philox draw (numpy vs the library's host export), the oracle's probabilities
against the reference's binary search, and argument validation of zl_sample / zl_llama_set_sampling."""
import ctypes

import numpy as np
import pytest

from tests import sampling_oracle as so


def test_philox_known_answer():
    # Random123 known-answer vector for philox4x32-10, counter 0, key 0
    out = so.philox4x32_10([0, 0, 0, 0], [0, 0])
    assert [int(w) for w in out] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


def test_philox_known_answer_all_ones():
    # Random123 known-answer vector: counter and key all 0xffffffff
    f = 0xFFFFFFFF
    out = so.philox4x32_10([f, f, f, f], [f, f])
    assert [int(w) for w in out] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def test_uniform_range():
    u = so.uniform(np.arange(1000, dtype=np.uint64), 7)
    assert u.min() > 0 and u.max() <= 1.0
    assert np.all(u * 2 ** 24 == np.round(u * 2 ** 24))


def test_host_uniform_matches_oracle(lib):
    rng = np.random.default_rng(0)
    seeds = rng.integers(0, 2 ** 63, size=10000, dtype=np.uint64)
    seeds[:10] = [0, 1, 2 ** 32, 2 ** 32 - 1, 2 ** 64 - 1, 0xDEADBEEF, 5, 6, 7, 8]
    counters = rng.integers(0, 2 ** 32, size=10000, dtype=np.uint64)
    counters[:5] = [0, 1, 2 ** 31, 2 ** 32 - 1, 100]
    want = so.uniform_r(seeds, counters)
    got = np.array([lib.zl_sample_uniform(int(s), int(c)) for s, c in zip(seeds, counters)], dtype=np.uint32)
    np.testing.assert_array_equal(got, want)


def _rows():
    rng = np.random.default_rng(1)
    rows = [
        np.array([2.0, 1.0, 0.5, -1.0, 3.0], dtype=np.float32),
        np.array([1.0, 1.0, 1.0, 0.0, 0.0, 1.0], dtype=np.float32),            # ties
        np.array([0.0, -np.inf, 1.0, -np.inf, 1.0, -2.0], dtype=np.float32),  # -inf and ties
        np.round(rng.normal(size=40) * 2).astype(np.float32) / 2,              # tie-heavy
        rng.normal(size=40).astype(np.float32) * 3,
    ]
    return rows


SETTINGS = [(1.0, 1.0, 0), (0.7, 1.0, 0), (1.0, 0.9, 0), (1.0, 0.5, 0), (1.0, 1.0, 3), (0.8, 0.6, 4),
            (1.3, 0.95, 2), (1.0, 1.0, 100), (2.0, 0.3, 0)]


@pytest.mark.parametrize("setting", SETTINGS)
def test_oracle_probs_equal_reference_search_measure(setting):
    """Each token's oracle probability is the measure of the u in (0, 1] that the reference's binary search maps to it."""
    T, top_p, top_k = setting
    n = 200000
    u = (np.arange(n) + 0.5) / n
    for l in _rows():
        p = so.probs(l, T, top_p, top_k)
        assert abs(p.sum() - 1) < 1e-12 and p.min() >= 0
        hits = np.bincount(so.reference_binary_search(l, T, top_p, top_k, u), minlength=len(l))
        np.testing.assert_allclose(hits / n, p, atol=2.0 / n + 1e-9)
        assert np.all(p[np.isneginf(l)] == 0)
        for uu in u[::997]:
            tok, amb = so.pick(l, T, top_p, top_k, uu)
            if not amb:
                assert tok == int(so.reference_binary_search(l, T, top_p, top_k, uu))
                assert p[tok] > 0


def test_oracle_greedy_and_fallback():
    l = np.array([1.0, 3.0, 3.0, -1.0], dtype=np.float32)
    assert so.pick(l, 0.0, 1.0, 0, 0.5) == (1, False)
    assert so.pick(l, 1.0, 1.0, 1, 0.5) == (1, False)
    inf_row = np.array([-np.inf, -np.inf], dtype=np.float32)
    assert so.pick(inf_row, 1.0, 1.0, 0, 0.5) == (0, False)
    pos_inf = np.array([0.0, np.inf, np.inf], dtype=np.float32)
    assert so.pick(pos_inf, 1.0, 1.0, 0, 0.5) == (1, False)


def test_penalties_follow_reference_rule():
    l = np.array([2.0, -2.0, 1.0, 0.0], dtype=np.float32)
    np.testing.assert_array_equal(so.penalise(l, [0, 1, 1], 2.0, 0.0), np.array([1.0, -4.0, 1.0, 0.0], np.float32))
    np.testing.assert_array_equal(so.penalise(l, [0, 3], 2.0, 0.5), np.array([1.5, -2.0, 1.0, -0.5], np.float32))


def test_bitmap_round_trip():
    h = so.history_bitmap([[0, 31, 32, 999], []], 1000)
    assert h.shape == (2, 32)
    assert so.bitmap_tokens(h[0], 1000) == {0, 31, 32, 999}
    assert so.bitmap_tokens(h[1], 1000) == set()


BAD = [dict(temperature=-0.5), dict(top_p=0.0), dict(top_p=1.5), dict(top_p=-0.1), dict(top_k=-1),
       dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(temperature=float("nan")),
       dict(presence_penalty=float("inf"))]


@pytest.mark.parametrize("bad", BAD, ids=[",".join("%s=%s" % kv for kv in b.items()) for b in BAD])
def test_bad_parameters_are_rejected(lib, bad):
    from zhilight_b200 import _lib
    p = _lib.sample_params(**bad)
    assert lib.zl_sample_check_params(ctypes.byref(p), 1) == _lib.ZLError(-1, "").code
    # zl_llama_set_sampling validates before it looks at the driver (so no GPU is needed to see the rejection)
    assert lib.zl_llama_set_sampling(None, 0, ctypes.byref(p)) == -1
    assert "invalid argument" in _lib.last_error()


def test_good_parameters_pass_check(lib):
    from zhilight_b200 import _lib
    arr = (_lib.SampleParams * 3)(_lib.sample_params(), _lib.sample_params(0.8, 0.95, 50, 1.2, 0.0, 3),
                                  _lib.sample_params(1.0, 1.0, 0, 1.0, -0.5, 2 ** 64 - 1))
    assert lib.zl_sample_check_params(ctypes.cast(arr, ctypes.c_void_p), 3) == 0


def test_zl_sample_rejects_bad_shapes(lib):
    from zhilight_b200 import _lib
    dummy = ctypes.c_void_p(16)   # never dereferenced: the checks run before any launch
    assert lib.zl_sample(None, 1, 10, dummy, None, None, None, 0, dummy, None, 0, 0, None) == -1
    assert lib.zl_sample(dummy, 0, 10, dummy, None, None, None, 0, dummy, None, 0, 0, None) == -1
    assert lib.zl_sample(dummy, 1, 0, dummy, None, None, None, 0, dummy, None, 0, 0, None) == -1
    assert lib.zl_sample(dummy, 1, 10, None, None, None, None, 0, dummy, None, 0, 0, None) == -1
    assert lib.zl_sample(dummy, 1, 100, dummy, None, None, dummy, 3, dummy, None, 0, 0, None) == -1   # history too short
    assert lib.zl_sample(dummy, 1, 262145, dummy, None, None, None, 0, dummy, None, 0, 0, None) == -2
    assert "unsupported" in _lib.last_error()
    assert lib.zl_sample_workspace_bytes(128, 128256) == 0


def test_header_exports_sampling(lib):
    from zhilight_b200 import _lib
    protos = _lib.protos()
    for name in ("zl_sample", "zl_sample_uniform", "zl_sample_workspace_bytes", "zl_sample_check_params",
                 "zl_llama_set_sampling"):
        assert name in protos
    assert ctypes.sizeof(_lib.SampleParams) == 32
