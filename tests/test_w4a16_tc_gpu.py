"""GPU parity: the wgmma W4A16 kernel (k_w4a16_ts: A operand in registers, ZLW4I layout) vs the CPU oracle.

The kernel rounds w = (q - z) * s to fp16 once (what the reference's M > 40 dequant + cuBLASLt route does,
q_gemm_k_major.cu:843-905, 1083-1100), multiplies fp16 x fp16 exactly and accumulates all of K in fp32.
Tolerance (north_star): relative L2 <= 1e-3 against the fp32 oracle for fp16 outputs."""
import numpy as np
import pytest
import torch

from oracle import gptq, ops as oops
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _dev(a, cuda):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _setup(cuda, k, n, sym, seed, row_map=None):
    from zhilight_b200 import ops
    qw, qz, sc, gi = gptq.make_gptq_checkpoint(k, n, 128, sym, seed=seed)
    o_qw, o_qz, o_sc, _ = gptq.to_k_major(qw, qz, sc, gi, 128)
    w = gptq.dequant_k_major_f32(o_qw, o_qz, o_sc, sym)
    packed = ops.w4_pack(_dev(o_qw.view(np.int32), cuda), _dev(o_qz, cuda), _dev(o_sc, cuda), 128, sym, row_map,
                         variant=1)
    return w, packed


@pytest.fixture
def splits(lib):
    yield lambda s: lib.zl_w4_tc_set_splits(s)
    lib.zl_w4_tc_set_splits(0)


def _check_watchdog(lib):
    assert lib.zl_w4_tc_watchdog() == 0


def test_route_selects_tcgen05(lib):
    assert lib.zl_w4_int_layout_route(1, 4096, 4096) == 3       # exact-integer mma.sync kernel
    assert lib.zl_w4_int_layout_route(4, 4096, 4096) == 3
    assert lib.zl_w4_int_layout_route(16, 512, 1024) == 3
    assert lib.zl_w4_int_layout_route(16, 4096, 4096) == 4      # 16 staged token rows of K = 4096 do not fit beside the rings
    assert lib.zl_w4_int_layout_route(17, 4096, 4096) == 4      # wgmma
    assert lib.zl_w4_int_layout_route(32, 4096, 14336) == 4
    assert lib.zl_w4_int_layout_route(8, 4096, 14336) == 4      # staged activations of the integer kernel do not fit
    assert lib.zl_w4_int_layout_route(2048, 6144, 4096) == 4
    assert lib.zl_w4_int_layout_route(32, 96, 4096) == 0        # N % 128 != 0: the fp16 mma.sync kernel (variant 0)


@pytest.mark.parametrize("m", [17, 32, 33, 64, 65, 128, 200, 256, 300])
def test_token_counts(lib, cuda, m):
    """every NTOK instantiation (32 / 64 / 128 / 256), ragged last 16-token chunk, and a second pass beyond 256"""
    from zhilight_b200 import ops
    k, n = 1024, 512
    w, packed = _setup(cuda, k, n, False, 5)
    x = torch.randn(m, k, generator=torch.Generator().manual_seed(m)).half()
    y = ops.w4a16_gemm_fused(x.to(cuda), packed, n, k, variant=1).float().cpu().numpy()
    _check_watchdog(lib)
    ref = gptq.gemm_f32(x.numpy(), w)
    assert rel_l2(y, ref) <= TOL
    for i in range(m):
        assert rel_l2(y[i], ref[i]) <= 2 * TOL, i


@pytest.mark.parametrize("k,n,m,sym", [(128, 128, 17, False), (256, 128, 32, True), (4096, 6144, 32, False),
                                        (4096, 4096, 24, True), (14336, 4096, 32, False), (14336, 4096, 5, False),
                                        (4096, 28672, 48, False), (8192, 1024, 128, False)])
def test_model_shapes(lib, cuda, k, n, m, sym):
    """Llama-3.1-8B / 70B-class projection shapes, asym and sym zeros, automatic k-split"""
    from zhilight_b200 import ops
    w, packed = _setup(cuda, k, n, sym, 3)
    x = torch.randn(m, k, generator=torch.Generator().manual_seed(1)).half()
    y = ops.w4a16_gemm_fused(x.to(cuda), packed, n, k, variant=1).float().cpu().numpy()
    _check_watchdog(lib)
    ref = gptq.gemm_f32(x.numpy(), w)
    assert rel_l2(y, ref) <= TOL


@pytest.mark.parametrize("s", [1, 2, 3, 4])
def test_split_k_is_deterministic_and_exact_enough(lib, cuda, splits, s):
    from zhilight_b200 import ops
    k, n, m = 2048, 256, 40
    w, packed = _setup(cuda, k, n, False, 8)
    x = torch.randn(m, k, generator=torch.Generator().manual_seed(2)).half().to(cuda)
    splits(s)
    y1 = ops.w4a16_gemm_fused(x, packed, n, k, variant=1)
    y2 = ops.w4a16_gemm_fused(x, packed, n, k, variant=1)
    _check_watchdog(lib)
    assert torch.equal(y1, y2)                                    # partials are reduced in split order
    assert rel_l2(y1.float().cpu().numpy(), gptq.gemm_f32(x.cpu().numpy(), w)) <= TOL


@pytest.mark.parametrize("m,s", [(20, 1), (40, 2)])
def test_bias_residual_swiglu(lib, cuda, splits, m, s):
    from zhilight_b200 import ops
    k, f = 1024, 1280
    rm = ops.swiglu_row_map(f, cuda)
    w, packed = _setup(cuda, k, 2 * f, False, 7, rm)
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(m, k, generator=g)).half()
    splits(s)
    y = ops.w4a16_gemm_fused(x.to(cuda), packed, 2 * f, k, epilogue=ops.EPI_SWIGLU, variant=1).float().cpu().numpy()
    _check_watchdog(lib)
    gu = oops._t(gptq.gemm_f32(x.numpy(), w), "f16")              # T(gate), T(up) like the reference's two GEMVs
    gate, up = gu[:, :f], gu[:, f:]
    ref = gate / (1.0 + np.exp(-gate)) * up
    assert rel_l2(y, ref) <= 2e-3
    # bias + residual on a plain projection
    n = 512
    w2, packed2 = _setup(cuda, k, n, True, 4)
    bias = (torch.randn(n, generator=g) * 0.5).half()
    res = torch.randn(m, n, generator=g).half()
    y2 = ops.w4a16_gemm_fused(x.to(cuda), packed2, n, k, bias=bias.to(cuda), residual=res.to(cuda),
                              epilogue=ops.EPI_RESIDUAL, variant=1).float().cpu().numpy()
    _check_watchdog(lib)
    lin = oops._t(gptq.gemm_f32(x.numpy(), w2) + bias.float().numpy(), "f16")
    ref2 = oops._t(lin + res.float().numpy(), "f16")
    assert rel_l2(y2, ref2) <= TOL


@pytest.mark.parametrize("d,hq,hkv,k,t,s", [(128, 4, 2, 512, 24, 0), (64, 4, 2, 256, 40, 0), (128, 8, 1, 1024, 130, 0),
                                           (128, 32, 8, 4096, 32, 0), (128, 32, 8, 4096, 20, 3), (128, 8, 2, 2048, 32, 2)])
def test_qkv_rope_epilogue(lib, cuda, splits, d, hq, hkv, k, t, s):
    """fused qkv split + RoPE + KV append vs the stand-alone rope/append operator on the plain GEMM output"""
    from zhilight_b200 import ops
    n = (hq + 2 * hkv) * d
    rm = ops.qkv_rope_row_map(hq + 2 * hkv, d, cuda)
    _, packed = _setup(cuda, k, n, False, 14, rm)
    _, packed_plain = _setup(cuda, k, n, False, 14)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(t, k, generator=g).half().to(cuda)
    pos = torch.tensor([(5 * i) % 61 for i in range(t)], dtype=torch.int32, device=cuda)
    cos, sin = ops.rope_cos_sin(pos, d, 10000.0)
    tb = torch.tensor([i % 3 for i in range(t)], dtype=torch.int32, device=cuda)
    pl = torch.tensor([i // 3 for i in range(t)], dtype=torch.int32, device=cuda)     # (task, slot) pairs are unique
    slots = t // 3 + 2
    kb = [torch.zeros(slots, hkv, d, dtype=torch.float16, device=cuda) for _ in range(3)]
    vb = [torch.zeros(slots, hkv, d, dtype=torch.float16, device=cuda) for _ in range(3)]
    splits(s)
    q = ops.w4a16_gemm_fused(x, packed, n, k, epilogue=ops.EPI_QKV_ROPE, variant=1,
                             rope=dict(cos=cos, sin=sin, token_batch=tb, placement=pl, k_bufs=kb, v_bufs=vb,
                                       num_heads=hq, num_kv_heads=hkv, dim_head=d))
    _check_watchdog(lib)
    splits(0)
    qkv = ops.w4a16_gemm_fused(x, packed_plain, n, k, variant=1)
    assert torch.isfinite(q).all() and torch.isfinite(qkv).all()
    kb2 = [torch.zeros_like(b) for b in kb]
    vb2 = [torch.zeros_like(b) for b in vb]
    q2 = ops.qkv_rope_append(cos, sin, qkv, tb, pl, kb2, vb2, hq, hkv, d)
    torch.testing.assert_close(q, q2, rtol=2 ** -9, atol=3e-3)
    for a, b in zip(kb + vb, kb2 + vb2):
        torch.testing.assert_close(a, b, rtol=2 ** -9, atol=3e-3)
    assert float(kb[0].abs().max()) > 0 and float(q.abs().max()) > 0


def test_strided_activations_and_fused_norm_is_rejected(lib, cuda):
    from zhilight_b200 import ops, _lib
    k, n, m = 512, 256, 20
    w, packed = _setup(cuda, k, n, False, 21)
    big = torch.randn(m, k + 64, generator=torch.Generator().manual_seed(3)).half().to(cuda)
    x = big[:, :k]                                                # ldx = k + 64
    y = ops.w4a16_gemm_fused(x, packed, n, k, variant=1).float().cpu().numpy()
    assert rel_l2(y, gptq.gemm_f32(x.cpu().numpy(), w)) <= TOL
    with pytest.raises(_lib.ZLError) as e:
        ops.w4a16_gemm_fused(x, packed, n, k, variant=1, ln_weight=torch.ones(k, dtype=torch.float16, device=cuda))
    assert e.value.code == -2


@pytest.mark.parametrize("m", [17, 32])
@pytest.mark.parametrize("tp_mode", [1, 2])
def test_tp_exchange_is_rejected_on_the_wgmma_route(lib, cuda, m, tp_mode):
    """Only the exact-integer kernel (M <= 16) carries the tensor-parallel exchange: a one-rank comm with opened state
    gets as far as that check."""
    import ctypes
    from zhilight_b200 import _lib, dist
    k, n = 512, 256
    _, packed = _setup(cuda, k, n, False, 21)
    assert lib.zl_w4_int_layout_route(m, n, k) == 4
    x = torch.randn(m, k, generator=torch.Generator().manual_seed(3)).half().to(cuda)
    y = torch.empty(m, n, dtype=torch.float16, device=cuda)
    h_out = torch.empty_like(x)
    comm = dist.TPComm(m * n, 0, 1)
    try:
        a = _lib.W4FusedArgs()
        a.x, a.ldx, a.packed, a.y, a.M, a.N, a.K, a.group_size, a.variant = (x.data_ptr(), k, packed.data_ptr(),
                                                                              y.data_ptr(), m, n, k, 128, 1)
        a.tp_mode, a.tp_comm, a.tp_h_out = tp_mode, comm.handle.value, h_out.data_ptr()
        assert lib.zl_w4a16_gemm_fused(ctypes.byref(a), None) == -2
    finally:
        comm.close()
