"""The L2 head a W4A16 GEMM prefetches for its successor (zl_w4_v3_l2_head, the same v3_head_ranges the integer kernel
runs): for each successor warp, the byte ranges of its first H ring items, checked against an independent restatement of
the kernel's producer order (issue_next in w4a16_gemm_v3.cu) over the Llama-3.1-8B decode shapes."""
import ctypes

import numpy as np
import pytest

from zhilight_b200 import _lib

BLOCK = 2128          # one ZLW4I record: 32 rows x 128 k
SMS = 132             # H100 SXM
# (N, K, tp_mode) of qkv, o, gate_up (fused), down: one GPU, and the shards of TP = 2 (reduce-in / push exchanges)
SHAPES = [(6144, 4096, 0), (4096, 4096, 0), (28672, 4096, 0), (4096, 14336, 0),
          (3072, 4096, 1), (4096, 2048, 2), (14336, 4096, 1), (4096, 7168, 2)]


@pytest.fixture(scope="module")
def lib():
    lb = _lib.load()
    lb.zl_w4_v3_plan.restype = ctypes.c_int
    lb.zl_w4_v3_l2_head.restype = ctypes.c_int
    return lb


def plan(lib, mc, N, K, tp):
    """(warps per sub-CTA, sub-CTAs, ring stages, grid, sub-major) of the integer kernel, or None where (mc, N, K) routes
    elsewhere"""
    out = (ctypes.c_int * 9)()
    rc = lib.zl_w4_v3_plan(mc, N, K, tp, SMS, out)
    # the plan exists exactly where the public router picks the integer kernel (its staged activations fit shared memory)
    assert (rc == 0) == (lib.zl_w4_int_layout_route(mc, N, K) == 3), (mc, N, K, rc)
    if rc != 0:
        assert rc == -2
        return None
    nt, warps, subs, stages, rt, pack, grid, smem, sub_major = list(out)
    return warps, subs, stages, grid, sub_major


def producer_items(N, K, warps, subs, grid, sub_major):
    """per warp of the launch (CTA-major, then sub-CTA, then warp): its ring items in producer order, as byte offsets.
    Sub-CTA `sub` of CTA `cta` starts at tile sub * grid + cta (sub-major) or cta * subs + sub, strides grid * subs."""
    G, n_tiles = K // 128, N // 32
    items = []
    for cta in range(grid):
        for sub in range(subs):
            for wl in range(warps):
                g_begin, g_end = wl * G // warps, (wl + 1) * G // warps
                seq = [(tile * G + g) * BLOCK
                       for tile in range(sub * grid + cta if sub_major else cta * subs + sub, n_tiles, grid * subs)
                       for g in range(g_begin, g_end)]
                items.append(seq)
    return items


def head(lib, mc, N, K, tp, H):
    cap = 1 << 16
    out = (ctypes.c_longlong * (3 * cap))()
    n = lib.zl_w4_v3_l2_head(mc, N, K, tp, SMS, H, out, cap)
    assert n >= 0
    return np.frombuffer(out, dtype=np.int64)[: 3 * n].reshape(n, 3)


@pytest.mark.parametrize("mc", [1, 2, 4, 8])
@pytest.mark.parametrize("N,K,tp", SHAPES)
@pytest.mark.parametrize("H", [1, 2, 4, 5])
def test_head_is_each_warps_first_ring_items(lib, mc, N, K, tp, H):
    pl = plan(lib, mc, N, K, tp)
    if pl is None:
        out = (ctypes.c_longlong * 3)()
        assert lib.zl_w4_v3_l2_head(mc, N, K, tp, SMS, H, out, 1) == -2
        return
    warps, subs, stages, grid, sub_major = pl
    blob = (N // 32) * (K // 128) * BLOCK
    rng = head(lib, mc, N, K, tp, H)
    # inside the blob, record-aligned, non-overlapping
    assert (rng[:, 1] % BLOCK == 0).all() and (rng[:, 2] % BLOCK == 0).all() and (rng[:, 2] > 0).all()
    assert (rng[:, 1] >= 0).all() and (rng[:, 1] + rng[:, 2] <= blob).all()
    order = np.argsort(rng[:, 1], kind="stable")
    starts, ends = rng[order, 1], rng[order, 1] + rng[order, 2]
    assert (starts[1:] >= ends[:-1]).all()
    # per warp: exactly the first min(H, total) items its producer requests, in that order
    items = producer_items(N, K, warps, subs, grid, sub_major)
    got = [[] for _ in items]
    for sw, off, nb in rng:
        got[sw].extend(range(off, off + nb, BLOCK))
    for sw, seq in enumerate(items):
        assert got[sw] == seq[:H], (sw, got[sw][:8], seq[:8])


@pytest.mark.parametrize("mc", [1, 2, 4, 8])
@pytest.mark.parametrize("N,K,tp", SHAPES)
def test_deep_head_covers_whole_blob(lib, mc, N, K, tp):
    pl = plan(lib, mc, N, K, tp)
    if pl is None:
        return
    warps, subs, stages, grid, sub_major = pl
    H = max(len(s) for s in producer_items(N, K, warps, subs, grid, sub_major))
    rng = head(lib, mc, N, K, tp, H)
    blob = (N // 32) * (K // 128) * BLOCK
    covered = np.zeros(blob // BLOCK, np.int32)
    for _, off, nb in rng:
        covered[off // BLOCK: (off + nb) // BLOCK] += 1
    assert (covered == 1).all()


def test_plan_matches_decode_variants(lib):
    """batch 1 on 132 SMs: wide GEMMs (N/32 > #SMs) run 2 x 8 warps with 5-stage rings on every SM in sub-major tile
    order, tall ones 1 x 16 with 4"""
    assert plan(lib, 1, 6144, 4096, 0) == (8, 2, 5, 132, 1)
    assert plan(lib, 1, 28672, 4096, 0) == (8, 2, 5, 132, 1)
    assert plan(lib, 1, 4096, 4096, 0) == (16, 1, 4, 128, 0)
    assert plan(lib, 1, 4096, 14336, 0) == (16, 1, 4, 128, 0)
    assert plan(lib, 1, 14336, 4096, 1) == (8, 2, 4, 132, 1)   # tensor-parallel exchange: 4-stage variants
    assert plan(lib, 4, 28672, 4096, 0) == (8, 2, 4, 132, 1)   # 5-stage rings no longer fit with 4 staged rows
    assert plan(lib, 8, 4096, 4096, 0) is None              # the wgmma kernel serves M = 8 at K = 4096
    assert plan(lib, 17, 4096, 4096, 0) is None
