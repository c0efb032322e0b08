"""W8A8 Linear (SURVEY 8-a8 Int8Linear, 8-a9 Fp8Linear) through the C-ABI against the oracle.

INT8 is integer work with a two-multiply fp32 epilogue: bit-exact.  FP8 quantisation codes are bit-exact; the fp8
GEMM accumulates in fp32 in a different order than cuBLASLt: <= 1e-3 rel (fp16) like the reference's own Linear
tests (tests/test_linear.py:48-86)."""
import numpy as np
import pytest
import torch

from oracle import ops as oracle
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu
DT = {"f16": torch.float16, "bf16": torch.bfloat16}


def _x(m, k, tag, seed=0, amp=1.5):
    r = np.random.default_rng(seed)
    return oracle._t(r.standard_normal((m, k)) * amp, tag)


def _dev(a, tag, cuda):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DT[tag]).to(cuda)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("m,k", [(1, 512), (7, 4096), (32, 14336), (40, 1024)])
def test_int8_quant_per_token_bit_exact(lib, cuda, tag, m, k):
    from zhilight_b200 import ops
    x = _x(m, k, tag, seed=m)
    if m > 1:
        x[m // 2] = 0                                           # all-zero token
    q, s = ops.int8_quant_per_token(_dev(x, tag, cuda))
    oq, os_ = oracle.int8_quant_per_token(x)
    np.testing.assert_array_equal(q.cpu().numpy(), oq)
    np.testing.assert_array_equal(s.cpu().numpy(), os_)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("m,n,k,f32_scale,with_bias", [
    (1, 4096, 4096, False, False), (3, 1000, 512, True, False), (8, 6144, 4096, False, True),
    (9, 4096, 14336, False, False), (16, 64, 64, False, True), (17, 2048, 2048, True, True),
    (32, 28672, 4096, False, False), (33, 1024, 1024, False, False), (70, 512, 256, False, True),
    # M > 32: the wgmma s8 kernel (both operands through tensor-TMA, s32 register accumulators, split-k)
    (64, 6144, 4096, False, True), (128, 4096, 14336, True, False), (300, 1000, 1024, False, True)])
def test_int8_linear_bit_exact(lib, cuda, tag, m, n, k, f32_scale, with_bias):
    from zhilight_b200 import ops
    r = np.random.default_rng(n + m)
    x = _x(m, k, tag, seed=k + m)
    w_q = r.integers(-127, 128, size=(n, k)).astype(np.int8)
    w_s = oracle._t(0.0005 + 0.003 * r.random(n), tag)
    bias = oracle._t(0.2 * r.standard_normal(n), tag) if with_bias else None
    ws_dev = torch.from_numpy(w_s).to(cuda) if f32_scale else _dev(w_s, tag, cuda)
    y = ops.int8_linear(_dev(x, tag, cuda), torch.from_numpy(w_q).to(cuda), ws_dev,
                        None if bias is None else _dev(bias, tag, cuda))
    ref = oracle.int8_linear(x, w_q, w_s, tag, bias)
    np.testing.assert_array_equal(y.float().cpu().numpy(), ref)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
def test_rmsnorm_quant(lib, cuda, tag):
    from zhilight_b200 import ops
    t, d = 6, 4096
    r = np.random.default_rng(5)
    x = _x(t, d, tag, seed=3)
    x[2] = 0
    w = oracle._t(1.0 + 0.2 * r.standard_normal(d), tag)
    for scale in (1.0, 2.5):
        y, q, qs = ops.rmsnorm_quant(_dev(x, tag, cuda), _dev(w, tag, cuda), 1e-5, scale)
        oy, oq, oqs = oracle.rmsnorm_quant(x, w, 1e-5, scale, tag)
        np.testing.assert_array_equal(q.cpu().numpy(), oq)
        np.testing.assert_allclose(qs.cpu().numpy(), oqs, rtol=2e-6)
        assert rel_l2(y.float().cpu().numpy(), oy) < (1e-3 if tag == "f16" else 4e-3)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("m,k", [(1, 4096), (5, 512), (32, 14336)])
def test_fp8_quant_codes_bit_exact(lib, cuda, tag, m, k):
    from zhilight_b200 import ops
    x = _x(m, k, tag, seed=11 + m, amp=3.0)
    q, s = ops.fp8_quant_per_tensor(_dev(x, tag, cuda))
    ov, os_ = oracle.fp8_quant_per_tensor(x, dtype=tag)
    assert s.item() == os_
    np.testing.assert_array_equal(oracle.e4m3_decode(q.cpu().numpy()), ov)


@pytest.mark.parametrize("tag", ["f16", "bf16"])
@pytest.mark.parametrize("m,n,k,with_bias", [(1, 4096, 4096, False), (4, 1000, 512, True), (16, 6144, 4096, False),
                                             (32, 4096, 14336, True), (35, 256, 128, False),
                                             # M > 32: the wgmma e4m3 kernel
                                             (64, 6144, 4096, True), (130, 4096, 4096, False)])
def test_fp8_linear(lib, cuda, tag, m, n, k, with_bias):
    from zhilight_b200 import ops
    r = np.random.default_rng(n)
    x = _x(m, k, tag, seed=k)
    w8 = r.integers(0, 256, size=(n, k)).astype(np.uint8)
    w8[(w8 & 0x7F) == 0x7F] = 0x30
    w8[(w8 & 0x78) > 0x50] &= 0xAF                               # keep |w| <= ~30 so fp16 outputs stay finite
    w_scale = np.float32(0.004)
    bias = oracle._t(0.2 * r.standard_normal(n), tag) if with_bias else None
    y = ops.fp8_linear(_dev(x, tag, cuda), torch.from_numpy(w8).to(cuda),
                       torch.tensor([w_scale], dtype=torch.float32, device=cuda),
                       None if bias is None else _dev(bias, tag, cuda))
    ref = oracle.fp8_linear(x, oracle.e4m3_decode(w8), w_scale, tag, bias)
    assert np.isfinite(ref).all()
    assert rel_l2(y.float().cpu().numpy(), ref) < (1e-3 if tag == "f16" else 4e-3)


def test_w8_argument_errors(lib, cuda):
    from zhilight_b200 import _lib, ops
    xq = torch.zeros((2, 96), dtype=torch.int8, device=cuda)          # K % 64 != 0
    sx = torch.ones(2, device=cuda)
    w = torch.zeros((16, 96), dtype=torch.int8, device=cuda)
    with pytest.raises(_lib.ZLError):
        ops.w8a8_gemm(xq, sx, w, torch.ones(16, device=cuda), torch.float16)
    with pytest.raises(_lib.ZLError):                                  # fp8 needs f32 scalar scales
        ops.w8a8_gemm(torch.zeros((2, 64), dtype=torch.uint8, device=cuda), sx,
                      torch.zeros((16, 64), dtype=torch.uint8, device=cuda),
                      torch.ones(1, dtype=torch.float16, device=cuda), torch.float16, kind=ops.W8_FP8)
