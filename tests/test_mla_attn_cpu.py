"""CPU-only checks of the MLA decode attention entry point: argument validation of zl_mla_decode_attention before any
CUDA call, its workspace formula, the shape checks of ops.mla_decode_attention, and the MLA oracle against the reference's
own kernels (tests/golden/mla_ref.npz)."""
import ctypes

import numpy as np
import pytest
import torch

from tests import mla_golden
from zhilight_b200 import _lib, ops

INVALID, UNSUPPORTED = -1, -2


def _call(lib, q=16, lens=16, kv=16, out=16, b=2, len_q=1, h=16, max_len=64, ws=0, ws_bytes=0, dtype=0):
    p = lambda x: ctypes.c_void_p(x) if x else None
    return lib.zl_mla_decode_attention(p(q), p(lens), p(kv), None, 0.1, max_len, p(out), b, len_q, h, p(ws), ws_bytes,
                                       dtype, 0, None)


def test_mla_attention_argument_checks(lib):
    assert _call(lib, q=0) == INVALID
    assert _call(lib, lens=0) == INVALID
    assert _call(lib, kv=0) == INVALID
    assert _call(lib, out=0) == INVALID
    assert _call(lib, b=0) == INVALID
    assert _call(lib, len_q=0) == INVALID
    assert _call(lib, max_len=0) == INVALID
    assert _call(lib, h=0) == INVALID
    assert _call(lib, h=129) == UNSUPPORTED
    assert _call(lib, dtype=2) == UNSUPPORTED
    # more than 256 keys may be split: the workspace is required and must be large enough
    need = lib.zl_mla_decode_attention_workspace_bytes(2, 1, 16, 4096)
    assert need > 0
    assert _call(lib, max_len=4096) == INVALID
    assert _call(lib, max_len=4096, ws=16, ws_bytes=need - 1) == INVALID


@pytest.mark.parametrize("b,len_q,h,max_len", [(1, 1, 16, 1), (1, 1, 16, 256), (1, 1, 16, 257), (3, 2, 128, 1025),
                                               (64, 1, 16, 16384), (2, 1, 1, 100000)])
def test_mla_workspace_formula(lib, b, len_q, h, max_len):
    splits = min(64, -(-max_len // 256))
    want = b * len_q * h * splits * (512 + 2) * 4 if splits > 1 else 0
    assert lib.zl_mla_decode_attention_workspace_bytes(b, len_q, h, max_len) == want
    assert lib.zl_mla_decode_attention_workspace_bytes(0, len_q, h, max_len) == 0


def test_mla_ops_reject_malformed_shapes(lib):
    q = torch.zeros(2, 1, 16, 576, dtype=torch.float16)
    kv = [torch.zeros(8, 576, dtype=torch.float16), torch.zeros(8, 1, 576, dtype=torch.float16)]
    lens = torch.tensor([8, 8], dtype=torch.int32)
    bad = [
        (torch.zeros(2, 1, 16, 512, dtype=torch.float16), kv),                     # q is not 576 wide
        (torch.zeros(2, 16, 576, dtype=torch.float16), kv),                        # q is not 4-d
        (q, [torch.zeros(8, 512, dtype=torch.float16)] * 2),                       # cache is not 576 wide
        (q, [torch.zeros(8, 2, 576, dtype=torch.float16)] * 2),                    # more than one latent head
        (q, kv[:1]),                                                               # one cache per task
        (q, [torch.zeros(8, 576, dtype=torch.bfloat16)] * 2),                      # cache dtype differs from q
    ]
    for qq, kk in bad:
        with pytest.raises(_lib.ZLError) as e:
            ops.mla_decode_attention(qq, lens, kk, None, 0.1, 8)
        assert e.value.code == -1


def test_mla_oracle_against_reference_fixture():
    """tests/golden/mla_ref.npz holds the reference's own MLA kernels' outputs on the case_mla inputs; they pin the oracle."""
    with np.load(mla_golden.FIXTURE) as g:
        assert sorted(g.files) == sorted(k for _, _, k in mla_golden.keys())
        errs = mla_golden.check(g)
    assert max(errs.values()) < 1e-4, errs


def test_mla_oracle_is_softmax_over_the_latent_rows():
    r = np.random.default_rng(3)
    kv = r.standard_normal((30, 1, 576)).astype(np.float32)
    q = r.standard_normal((1, 1, 4, 576)).astype(np.float32)
    out = mla_golden.mla_oracle(q, [kv], [30], [np.ones((1, 30), np.int8)], 0.05, "f32")
    assert out.shape == (1, 1, 4, 512)
    logit = (kv[:, 0] @ q[0, 0, 2]) * np.float32(0.05)
    p = np.exp(logit - logit.max())
    np.testing.assert_allclose(out[0, 0, 2], (p / p.sum()) @ kv[:, 0, :512], rtol=2e-5, atol=2e-6)
