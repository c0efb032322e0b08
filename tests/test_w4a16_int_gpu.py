"""GPU parity: the exact-integer W4A16 kernel (ZLW4I layout, IMMA) vs the CPU oracle.

The kernel decomposes activations into 16-bit block-floating-point integers per 128-group and accumulates
q*m exactly in int32, so it must be at least as close to the fp32 oracle as the fp16-MMA path."""
import numpy as np
import pytest
import torch

from oracle import gptq, ops as oops
from tests.helpers import rel_l2, w4i_pack_numpy

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _dev(a, cuda):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _setup(cuda, k, n, sym, seed, row_map=None):
    from zhilight_b200 import ops
    qw, qz, sc, gi = gptq.make_gptq_checkpoint(k, n, 128, sym, seed=seed)
    o_qw, o_qz, o_sc, _ = gptq.to_k_major(qw, qz, sc, gi, 128)
    w = gptq.dequant_k_major_f32(o_qw, o_qz, o_sc, sym)
    args = (_dev(o_qw.view(np.int32), cuda), _dev(o_qz, cuda), _dev(o_sc, cuda), 128, sym, row_map)
    return w, ops.w4_pack(*args, variant=1), ops.w4_pack(*args, variant=0), (o_qw, o_qz, o_sc)


@pytest.mark.parametrize("k,n,sym", [(128, 32, False), (512, 64, True), (4096, 256, False)])
def test_int_layout_bit_exact_and_roundtrip(lib, cuda, k, n, sym):
    from zhilight_b200 import ops
    w, packed_i, _, (o_qw, o_qz, o_sc) = _setup(cuda, k, n, sym, 3)
    np.testing.assert_array_equal(packed_i.cpu().numpy(), w4i_pack_numpy(o_qw, o_qz, o_sc, sym))
    r_qw, r_qz, r_sc = ops.w4_unpack(packed_i, n, k, variant=1)
    np.testing.assert_array_equal(r_qw.cpu().numpy().view(np.uint32), o_qw)
    np.testing.assert_array_equal(r_qz.cpu().numpy(), np.full_like(o_qz, 8) if sym else o_qz)
    np.testing.assert_array_equal(r_sc.cpu().numpy(), o_sc)


@pytest.mark.parametrize("sym", [False, True])
def test_config1_1x4096x4096_int(lib, cuda, sym):
    from zhilight_b200 import ops
    k = n = 4096
    w, packed_i, packed_h, _ = _setup(cuda, k, n, sym, 0)
    x = torch.randn(1, k, generator=torch.Generator().manual_seed(0)).half()
    y = ops.w4a16_gemm_fused(x.to(cuda), packed_i, n, k, variant=1).float().cpu().numpy()
    ref = gptq.gemm_f32(x.numpy(), w)
    assert rel_l2(y, ref) <= TOL
    y_h = ops.w4a16_gemm(x.to(cuda), packed_h, n, k).float().cpu().numpy()
    assert rel_l2(y, y_h) <= TOL
    # integer accumulation is exact: the only error left is the fp16 rounding of the output
    assert rel_l2(y, ref) <= 4e-4


@pytest.mark.parametrize("m", [1, 2, 3, 5, 8, 12, 16])
@pytest.mark.parametrize("k,n", [(1024, 512), (4096, 6144), (14336, 4096), (4096, 4096), (4096 + 128, 96), (256, 64), (256, 512)])
def test_shapes_and_batches_int(lib, cuda, m, k, n):
    from zhilight_b200 import ops, _lib
    route = _lib.load().zl_w4_int_layout_route(m, n, k)
    if route == 0:     # neither the integer kernel (staging too large) nor the wgmma kernel (N % 128): variant 0 territory
        with pytest.raises(_lib.ZLError):
            w, packed_i, _, _ = _setup(cuda, k, n, False, 5)
            ops.w4a16_gemm_fused(torch.zeros(m, k, dtype=torch.float16, device=cuda), packed_i, n, k, variant=1)
        return
    # route 3: exact-integer kernel; route 4: the same ZLW4I weights through the wgmma kernel (fp16-rounded weights)
    w, packed_i, _, _ = _setup(cuda, k, n, False, 5)
    g = torch.Generator().manual_seed(m)
    x = (torch.randn(m, k, generator=g) * torch.logspace(-2, 1, k)[torch.randperm(k, generator=g)]).half()
    y = ops.w4a16_gemm_fused(x.to(cuda), packed_i, n, k, variant=1).float().cpu().numpy()
    ref = gptq.gemm_f32(x.numpy(), w)
    assert rel_l2(y, ref) <= TOL
    for i in range(m):
        assert rel_l2(y[i], ref[i]) <= 2 * TOL


def test_edge_activations_int(lib, cuda):
    """all-zero groups, huge / tiny magnitudes, negative extremes: the block exponent logic must hold."""
    from zhilight_b200 import ops
    k, n = 512, 64
    w, packed_i, _, _ = _setup(cuda, k, n, False, 6)
    x = torch.zeros(4, k, dtype=torch.float16)
    x[0, 128:256] = 60000.0
    x[0, 256] = -65504.0
    x[1, :] = 6e-5
    x[1, 5] = -6.1e-5
    x[2, 300:] = torch.randn(k - 300).half() * 1e-3
    x[3] = torch.randn(k).half()
    x[3, 0] = 1000.0
    y = ops.w4a16_gemm_fused(x.to(cuda), packed_i, n, k, variant=1).float().cpu().numpy()
    ref = oops._t(gptq.gemm_f32(x.numpy(), w), "f16")
    finite = np.isfinite(ref)
    assert np.isfinite(y[finite]).all()
    for i in range(4):
        f = finite[i]
        assert rel_l2(y[i][f], ref[i][f]) <= 2e-3, i


@pytest.mark.parametrize("m", [2, 6, 12])
def test_nonfinite_activations_propagate_int(lib, cuda, m):
    """Inf / NaN in the activations: the reference GEMV (q_gemm_k_major.cu:127-173) multiplies them through and every
    output of that token becomes NaN or +-Inf.  The integer decomposition cannot carry them, so the kernel poisons the
    token's outputs with NaN -- the non-finite pattern must equal the fp32 oracle's, and other tokens stay exact."""
    from zhilight_b200 import ops
    k, n = 512, 96
    w, packed_i, _, _ = _setup(cuda, k, n, False, 11)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(m, k, generator=g).half()
    x[0, 7] = float("inf")
    x[1, 300] = float("nan")
    if m > 2:
        x[2, 130] = float("-inf")
        x[2, 131] = float("inf")
    y = ops.w4a16_gemm_fused(x.to(cuda), packed_i, n, k, variant=1).float().cpu().numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        ref = gptq.gemm_f32(x.numpy(), w)
    bad_rows = [0, 1] + ([2] if m > 2 else [])
    for i in range(m):
        if i in bad_rows:
            assert not np.isfinite(ref[i]).any(), i           # oracle: Inf * w is +-Inf (NaN where w == 0), NaN stays NaN
            assert not np.isfinite(y[i]).any(), i             # ours: the whole token is poisoned
        else:
            assert np.isfinite(y[i]).all()
            assert rel_l2(y[i], ref[i]) <= TOL
    # fused RMSNorm prologue: Inf * rsqrt(Inf) is NaN in the reference's layernorm too (layernorm.cu:9-42)
    lw = torch.ones(k).half()
    y2 = ops.w4a16_gemm_fused(x.to(cuda), packed_i, n, k, variant=1, ln_weight=lw.to(cuda)).float().cpu().numpy()
    for i in bad_rows:
        assert not np.isfinite(y2[i]).any(), i


@pytest.mark.parametrize("m", [1, 3])
def test_epilogues_and_fused_norm_int(lib, cuda, m):
    from zhilight_b200 import ops
    k, f = 1024, 5120
    rm = ops.swiglu_row_map(f, cuda)
    w, packed_i, _, _ = _setup(cuda, k, 2 * f, False, 7, rm)
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(m, k, generator=g) * 2.0).half()
    lw = (1 + 0.1 * torch.randn(k, generator=g)).half()
    y = ops.w4a16_gemm_fused(x.to(cuda), packed_i, 2 * f, k, epilogue=ops.EPI_SWIGLU, ln_weight=lw.to(cuda), eps=1e-5,
                             variant=1).float().cpu().numpy()
    xn = oops.rmsnorm(x.numpy(), lw.numpy(), 1e-5, 1.0, "f16")
    full = gptq.gemm_f32(xn, w)
    assert rel_l2(y, oops.silu_mul(full[:, :f], full[:, f:], "f16")) <= 2 * TOL
    # residual + bias on a "tall" shape (few tiles, large K)
    k2, n2 = 4096, 256
    w2, p2, _, _ = _setup(cuda, k2, n2, True, 8)
    x2 = torch.randn(m, k2, generator=g).half()
    bias = torch.randn(n2, generator=g).half()
    res = torch.randn(m, n2, generator=g).half()
    y2 = ops.w4a16_gemm_fused(x2.to(cuda), p2, n2, k2, bias=bias.to(cuda), residual=res.to(cuda),
                              epilogue=ops.EPI_RESIDUAL, variant=1).float().cpu().numpy()
    ref2 = oops.residual_add(oops._t(gptq.gemm_f32(x2.numpy(), w2, bias.numpy()), "f16"), res.numpy(), "f16")
    assert rel_l2(y2, ref2) <= TOL


@pytest.mark.parametrize("d,hq,hkv,k,t", [(128, 4, 2, 512, 3), (64, 4, 2, 256, 3), (64, 4, 2, 256, 16), (128, 4, 1, 512, 12),
                                          (64, 2, 1, 256, 4)])
def test_qkv_rope_epilogue_int(lib, cuda, d, hq, hkv, k, t):
    """Batch sizes of every kernel variant (digit-packed <= 4, NT=1 <= 8, NT=2 <= 16) x both head sizes."""
    from zhilight_b200 import ops
    n = (hq + 2 * hkv) * d
    rm = ops.qkv_rope_row_map(hq + 2 * hkv, d, cuda)
    w, packed_i, _, _ = _setup(cuda, k, n, False, 14, rm)
    _, _, packed_plain, _ = _setup(cuda, k, n, False, 14)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(t, k, generator=g).half().to(cuda)
    pos = torch.tensor([(5 * i) % 11 for i in range(t)], dtype=torch.int32, device=cuda)
    cos, sin = ops.rope_cos_sin(pos, d, 10000.0)
    tb = torch.tensor([i % 3 for i in range(t)], dtype=torch.int32, device=cuda)
    pl = torch.tensor([i // 3 for i in range(t)], dtype=torch.int32, device=cuda)     # (task, slot) pairs are unique
    kb = [torch.zeros(12, hkv, d, dtype=torch.float16, device=cuda) for _ in range(3)]
    vb = [torch.zeros(12, hkv, d, dtype=torch.float16, device=cuda) for _ in range(3)]
    q = ops.w4a16_gemm_fused(x, packed_i, n, k, epilogue=ops.EPI_QKV_ROPE, variant=1,
                             rope=dict(cos=cos, sin=sin, token_batch=tb, placement=pl, k_bufs=kb, v_bufs=vb,
                                       num_heads=hq, num_kv_heads=hkv, dim_head=d))
    qkv = ops.w4a16_gemm(x, packed_plain, n, k)
    kb2 = [torch.zeros_like(b) for b in kb]
    vb2 = [torch.zeros_like(b) for b in vb]
    q2 = ops.qkv_rope_append(cos, sin, qkv, tb, pl, kb2, vb2, hq, hkv, d)
    torch.testing.assert_close(q, q2, rtol=2 ** -9, atol=3e-3)
    for a, b in zip(kb + vb, kb2 + vb2):
        torch.testing.assert_close(a, b, rtol=2 ** -9, atol=3e-3)
