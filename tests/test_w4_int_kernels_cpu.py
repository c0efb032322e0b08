"""CPU checks of the exact-integer W4A16 kernel tests: the float64 oracle (tests/w4_int_oracle.py) against the exact GEMM,
including versions of it broken on purpose, and the coverage of every compiled kernel by the GPU cases
(tests/w4_int_cases.py), planned by the built library's own zl_w4_v3_plan."""
import ctypes

import numpy as np
import pytest

from tests import w4_int_cases as C
from tests import w4_int_oracle as O


# ---------------------------------------------------------------- the oracle
def _check_bound(r):
    ok = ~r["poison"]
    slack = 1e-12 * (np.abs(r["exact"]) + r["qb"] + 1)
    return bool((np.abs(r["v"] - r["exact"])[ok] <= (r["qb"] + slack)[ok]).all())


@pytest.mark.parametrize("pack", [False, True])
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("kind", ["rand", "adv", "headroom"])
def test_emulation_within_its_bound_of_the_exact_gemm(pack, norm, kind):
    n, k, m = 64, 896, 6
    q, z, s = C.weights(n, k, False, headroom=kind == "headroom", seed=1)
    x = C.activations(kind, m, k, seed=2)
    rng = np.random.default_rng(3)
    ln_w = (1 + 0.1 * rng.standard_normal(k)).astype(np.float16) if norm else None
    for k_perm in (None, rng.permutation(k)):
        r = O.gemm(x, q, z, s, pack=pack, ln_w=ln_w, k_perm=k_perm, bias=rng.standard_normal(n).astype(np.float16))
        assert _check_bound(r)
        assert (r["qb"] > 0).any() and np.isfinite(r["v"]).all()


def test_poisoned_tokens():
    q, z, s = C.weights(32, 512, False, seed=4)
    r = O.gemm(C.activations("nonfinite", 3, 512, seed=5), q, z, s, pack=False)
    assert list(r["poison"]) == [True, True, False]
    assert _check_bound(r)


def _representable(m, k, seed):
    """activations that are exactly m * 2^e: 11-bit integers times 2^(j - 10), the group maximum in binade j"""
    rng = np.random.default_rng(seed)
    x = np.zeros((m, k))
    for t in range(m):
        for g in range(k // 128):
            j = int(rng.integers(-6, 6))
            v = rng.integers(-1023, 1024, 128).astype(np.float64)
            v[rng.integers(128)] = 1024 + rng.integers(0, 1024)
            x[t, g * 128:(g + 1) * 128] = v * 2.0 ** (j - 10)
    return x.astype(np.float16)


@pytest.mark.parametrize("pack", [False, True])
def test_emulation_is_exact_on_representable_activations(pack):
    q, z, s = C.weights(96, 1024, False, seed=6)
    r = O.gemm(_representable(5, 1024, 7), q, z, s, pack=pack, bias=np.ones(96, np.float16))
    assert np.array_equal(r["v"], r["exact"])


def _tie_data(m, k, shift, seed):
    """groups with maximum 2^j whose other elements are (4 i + 1) 2^(j - shift), positive: with a mantissa step of
    2^(j - shift + 1) every one of them is a tie that rounds to even, i.e. down by 2^(j - shift)"""
    rng = np.random.default_rng(seed)
    x = np.zeros((m, k))
    for t in range(m):
        for g in range(k // 128):
            j = int(rng.integers(-4, 4))
            v = (4 * rng.integers(0, 16, 128) + 1) * 2.0 ** (j - shift)
            v[0] = 2.0 ** j
            x[t, g * 128:(g + 1) * 128] = v
    return x.astype(np.float16)


@pytest.mark.parametrize("pack", [False, True])
def test_broken_oracles_fail(pack):
    """kE one too small (a step twice the kernel's) or a dropped group break the bound check; kE one too large differs
    from the kernel's rounding by more than the GPU tolerance of one fp16 ulp"""
    n, k = 64, 1024
    q, z, s = C.weights(n, k, False, seed=8)
    z[:] = 0
    ke = O.KE_PACK if pack else O.KE
    x = _tie_data(4, k, ke, 9)                 # multiples of the kernel's step: its emulation is exact
    good = O.gemm(x, q, z, s, pack=pack)
    assert _check_bound(good) and np.array_equal(good["v"], good["exact"])
    for broken in (O.gemm(x, q, z, s, pack=pack, ke=ke - 1), O.gemm(x, q, z, s, pack=pack, drop_group=3)):
        broken["qb"] = good["qb"]
        assert not _check_bound(broken)
    x = _tie_data(4, k, ke + 1, 10)            # ties at the kernel's step
    kern = O.gemm(x, q, z, s, pack=pack)
    fine = O.gemm(x, q, z, s, pack=pack, ke=ke + 1)
    assert _check_bound(kern) and np.array_equal(fine["v"], fine["exact"])
    _, tol = O.epi_none(kern["v"], kern["f32"])
    assert (np.abs(fine["v"] - kern["v"]) > tol).all()


def test_pack_k_major_inverts_unpack():
    from oracle import gptq
    q = np.random.default_rng(0).integers(0, 16, size=(8, 256), dtype=np.uint8)
    assert np.array_equal(gptq.unpack_k_major(O.pack_k_major(q)), q)


# ---------------------------------------------------------------- the kernel table and the coverage of the GPU cases
@pytest.fixture(scope="module")
def lb():
    from zhilight_b200 import _lib
    return _lib.load()


def _plan(lb, mc, n, k, tp, sms=C.SMS):
    out = (ctypes.c_int * 9)()
    rc = lb.zl_w4_v3_plan(mc, n, k, tp, sms, out)
    return C.shape_of(out) if rc == 0 else None


def test_every_plan_is_a_compiled_shape(lb):
    """over mc 1..16, K 128..16384 and decode widths, the planner only returns shapes of the kernel table (shape_of raises
    otherwise), and never a tall (16-warp) one for 9..16 tokens"""
    seen = set()
    for tp in (0, 1, 2):
        for sms in (132, 114):
            for mc in range(1, 17):
                for k in range(128, 16384 + 1, 128):
                    for n in (1024, 2048, 4096, 4224, 4256, 6144, 14336, 28672):
                        sh = _plan(lb, mc, n, k, tp, sms)
                        if sh is not None:
                            seen.add((sh, tp != 0))
                            assert (C.SHAPES[sh][0] == 2) == (mc > 8)
    assert {sh for sh, tp in seen if not tp} == set(range(len(C.SHAPES)))
    assert {sh for sh, tp in seen if tp} == {i for i, s in enumerate(C.SHAPES) if s[3] == 4}


def coverage(lb):
    """(shape, NORM, fusion) -> number of GPU launches that run it, and shape -> epilogues seen at tp_mode 0"""
    hits = {kn: 0 for kn in C.kernels()}
    epis = {i: set() for i in range(len(C.SHAPES))}
    for mc, n, k, epi, norm, fu, sym, kind in C.CASES:
        sh = _plan(lb, mc, n, k, 0)
        assert sh is not None, (mc, n, k)
        assert fu != 2 or epi == "qkv"
        hits[(sh, norm, fu)] += 1
        epis[sh].add(epi)
        if fu == 2:                   # the int8 cache is checked against the same launch with the fp16 epilogue
            hits[(sh, norm, 0)] += 1
    for mc, n, k in C.TP_CASES:
        for norm in (0, 1):
            hits[(_plan(lb, mc, n, k, 2), norm, 5)] += 1
            for kv8 in (0, 1):
                hits[(_plan(lb, mc, n, k, 1), norm, C.fusion(1, None, kv8))] += 1
    return hits, epis


def test_gpu_cases_reach_every_kernel(lb):
    hits, epis = coverage(lb)
    assert len(hits) == 72
    missed = [(C.SHAPES[sh], norm, C.FUSIONS[f]) for (sh, norm, f), c in hits.items() if c == 0]
    assert not missed, missed
    for sh, seen in epis.items():
        assert seen == {"none", "res", "swiglu", "qkv"}, (C.SHAPES[sh], seen)


def test_gpu_cases_reach_the_shape_edges(lb):
    """each shape at both ends of its token range (where the planner lets it run there), with fewer groups than warps
    where it has 8 warps, a group count that is not a multiple of its warps, and more tiles than sub-CTAs"""
    by_shape = {}
    for mc, n, k, *_ in C.CASES:
        by_shape.setdefault(_plan(lb, mc, n, k, 0), []).append((mc, n, k))
    for sh, cases in by_shape.items():
        nt, warps, subs, stages, pack = C.SHAPES[sh]
        mcs = {c[0] for c in cases}
        lo, hi = (1, 4) if pack else (5, 8) if nt == 1 else (9, 16)
        if warps == 16 and not pack:
            hi = 7            # tall, K >= 4096: 8 staged rows no longer fit
        assert lo in mcs and hi in mcs, (C.SHAPES[sh], sorted(mcs))
        assert any((k // 128) % warps for _, _, k in cases), C.SHAPES[sh]
        if warps == 8 and (stages == 5 or nt == 2):   # the 4-stage NT = 1 shapes run at tp_mode 0 only where K is large
            assert any(k // 128 < warps for _, _, k in cases), C.SHAPES[sh]
        if warps == 8:
            assert any(n // 32 > C.SMS * subs for _, n, _ in cases), C.SHAPES[sh]
            assert any(C.SMS < n // 32 < 2 * C.SMS for _, n, _ in cases), C.SHAPES[sh]
