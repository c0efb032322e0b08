"""CPU-only checks of the joined-step attention and driver entry points: argument validation of zl_varlen_attention
before any CUDA call, its workspace formula, and the Python-side packing / validation of step_joined segments."""
import ctypes

import numpy as np
import pytest

from zhilight_b200.llama import pack_joined_segments

INVALID, UNSUPPORTED = -1, -2


def _call(lib, q=16, seg=16, nseg=1, rows=1, k=16, v=16, out=16, hq=32, hkv=8, d=128, max_keys=64, dtype=0):
    p = lambda x: ctypes.c_void_p(x) if x else None
    return lib.zl_varlen_attention(p(q), p(seg), nseg, rows, p(k), p(v), 0.125, max_keys, p(out), hq, hkv, d, None, 0,
                                   dtype, 0, None)


def test_varlen_attention_argument_checks(lib):
    # null pointers
    assert _call(lib, q=0) == INVALID
    assert _call(lib, seg=0) == INVALID
    assert _call(lib, k=0) == INVALID
    assert _call(lib, v=0) == INVALID
    assert _call(lib, out=0) == INVALID
    # nseg / rows mismatch: every segment holds at least one row
    assert _call(lib, nseg=3, rows=2) == INVALID
    assert _call(lib, nseg=0, rows=2) == INVALID
    assert _call(lib, rows=0) == INVALID
    assert _call(lib, max_keys=0) == INVALID
    # heads
    assert _call(lib, hq=30, hkv=8) == INVALID
    assert _call(lib, hkv=0) == INVALID
    # head dims and dtypes the kernel is not built for
    assert _call(lib, d=96) == UNSUPPORTED
    assert _call(lib, d=256) == UNSUPPORTED
    assert _call(lib, dtype=2) == UNSUPPORTED
    # the segment table is read as int4
    assert _call(lib, seg=20) == INVALID
    # more than one split needs the workspace
    assert _call(lib, max_keys=513) == INVALID


@pytest.mark.parametrize("rows,nseg,hq,d,max_keys", [(1, 1, 32, 128, 1), (512, 3, 32, 128, 4608), (40, 40, 8, 64, 513),
                                                     (16, 1, 64, 128, 512), (7, 2, 4, 64, 70000)])
def test_varlen_workspace_formula(lib, rows, nseg, hq, d, max_keys):
    lib.zl_varlen_attention_workspace_bytes.restype = ctypes.c_size_t
    splits = -(-max_keys // 512)
    want = rows * hq * splits * (d + 2) * 4 if splits > 1 else 0
    assert lib.zl_varlen_attention_workspace_bytes(rows, nseg, hq, d, max_keys) == want


def test_varlen_workspace_rejects_bad_sizes(lib):
    for args in [(0, 1, 32, 128, 600), (4, 0, 32, 128, 600), (4, 5, 32, 128, 600), (4, 1, 0, 128, 600),
                 (4, 1, 32, 128, 0)]:
        assert lib.zl_varlen_attention_workspace_bytes(*args) == 0


def test_pack_joined_segments():
    toks, seg = pack_joined_segments([(2, [5, 6, 7], 10, True), (0, np.array([9]), 4, False)], 4, 64, 100)
    np.testing.assert_array_equal(toks, [5, 6, 7, 9])
    np.testing.assert_array_equal(seg, [[2, 10, 3, 1], [0, 4, 1, 0]])
    assert toks.dtype == np.int32 and seg.dtype == np.int32


@pytest.mark.parametrize("segments", [
    [],                                              # nothing to run
    [(0, [1], 0, True)] * 2,                         # duplicate task
    [(4, [1], 0, True)],                             # task out of range
    [(-1, [1], 0, True)],
    [(0, [], 0, True)],                              # n < 1
    [(0, [[1, 2]], 0, True)],                        # tokens not 1-D
    [(0, [1.5], 0, True)],                           # tokens not integers
    [(0, [1], -1, True)],                            # pos0 < 0
    [(0, [1, 2], 63, True)],                         # pos0 + n > max_seq
    [(0, [100], 0, True)],                           # token out of range
    [(0, [-1], 0, True)],
    [(0, [1], 0)],                                   # not a 4-tuple
    [(t, [1], 0, True) for t in range(5)],           # more segments than max_batch
])
def test_pack_joined_segments_rejects(segments):
    with pytest.raises(ValueError):
        pack_joined_segments(segments, 4, 64, 100)
