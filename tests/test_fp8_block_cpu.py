"""CPU checks of the FP8 block-scaled Linear (QuantType 10): the oracle against the reference's own Python statement of
per_token_cast_to_fp8 (fp8_util.cu:298-304, run through torch's e4m3 cast), the block GEMM oracle against a dequantise-
then-matmul restatement, and the argument / configuration checks of the C-ABI, layers.Linear and the decode driver,
none of which needs a GPU."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ops
from tests import fp8_block_oracle as fb


def _torch_per_token_cast(x):
    """The reference's Python form (fp8_util.cu:298-304) on CPU tensors."""
    m, n = x.shape
    xv = x.view(m, -1, 128)
    amax = xv.abs().float().amax(dim=2).view(m, -1).clamp(1e-4)
    q = (xv.float() * (448.0 / amax.unsqueeze(2))).to(torch.float8_e4m3fn).view(m, n)
    return q.view(torch.uint8).numpy(), (amax / 448.0).view(m, -1).numpy()


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_quant_oracle_matches_reference_python(dt):
    rng = np.random.default_rng(1)
    m, k = 7, 512
    x = torch.from_numpy(rng.standard_normal((m, k)).astype(np.float32) * 3).to(dt)
    x[2, 128:256] = 0                                     # an all-zero group: amax clamps to 1e-4
    x[3, :128] = 0
    x[3, 5] = -7.5                                        # the group's extreme lands on -448
    x[4, 256:384] *= 1e-3                                 # tiny group
    q, s = fb.quant_per_token_group(x.float().numpy())
    tq, ts = _torch_per_token_cast(x)
    np.testing.assert_array_equal(q, tq)
    assert s.shape == (k // 128, 8)
    np.testing.assert_array_equal(s[:, :m].T, ts)
    assert q[3, 5] == 0xFE                                # -448
    assert (q[2, 128:256] == 0).all() and s[1, 2] == np.float32(1e-4) / np.float32(448)


def test_e4m3_encode_round_trips_every_code():
    codes = np.array([c for c in range(256) if (c & 0x7F) != 0x7F], np.uint8)
    vals = ops.e4m3_decode(codes)
    np.testing.assert_array_equal(fb.e4m3_encode(vals), codes)
    assert fb.e4m3_encode(np.array([1000.0, -1000.0], np.float32)).tolist() == [0x7E, 0xFE]   # satfinite


@pytest.mark.parametrize("n", [128, 200, 384])
def test_block_gemm_oracle_is_dequantised_matmul(n):
    rng = np.random.default_rng(n)
    m, k = 5, 384
    x = rng.standard_normal((m, k)).astype(np.float32)
    xq, sx = fb.quant_per_token_group(x)
    wq, sw = fb.random_weight(n, k, rng)
    y = fb.block_gemm(xq, sx, wq, sw)
    xd = ops.e4m3_decode(xq).astype(np.float64) * np.repeat(sx[:, :m].T, 128, axis=1)
    wd = fb.dequant_weight(wq, sw).astype(np.float64)
    ref = xd @ wd.T
    assert np.abs(y - ref).max() <= 1e-5 * np.abs(ref).max()
    # one scale per row (the first block's) is far off with scales spread over 1e-3 .. 1e2
    wrong = xd @ (ops.e4m3_decode(wq).astype(np.float64) * sw[np.arange(n) // 128, :1]).T
    assert np.linalg.norm(wrong - ref) > 0.1 * np.linalg.norm(ref)


def test_abi_rejects_bad_arguments(lib):
    p = ctypes.c_void_p(256)
    f = ctypes.c_void_p(256)
    # K % 128 != 0 is unsupported; null pointers, a scale leading dimension < M and bad dtypes are invalid
    assert lib.zl_fp8_quant_per_token_group(p, 192, p, f, 4, 4, 192, 0, 0, None) == -2
    assert lib.zl_fp8_quant_per_token_group(None, 256, p, f, 4, 4, 256, 0, 0, None) == -1
    assert lib.zl_fp8_quant_per_token_group(p, 256, p, f, 3, 4, 256, 0, 0, None) == -1
    assert lib.zl_fp8_quant_per_token_group(p, 256, p, f, 4, 4, 256, 2, 0, None) == -1
    assert lib.zl_fp8_quant_per_token_group(p, 128, p, f, 4, 4, 256, 0, 0, None) == -1        # ldx < K
    assert lib.zl_fp8_block_gemm(p, f, 4, p, f, p, 4, 256, 192, 0, 0, None) == -2
    assert lib.zl_fp8_block_gemm(p, None, 4, p, f, p, 4, 256, 256, 0, 0, None) == -1
    assert lib.zl_fp8_block_gemm(p, f, 4, None, f, p, 4, 256, 256, 0, 0, None) == -1
    assert lib.zl_fp8_block_gemm(p, f, 4, p, None, p, 4, 256, 256, 0, 0, None) == -1
    assert lib.zl_fp8_block_gemm(p, f, 2, p, f, p, 4, 256, 256, 0, 0, None) == -1              # x_scale_ld < M
    assert lib.zl_fp8_block_gemm(p, f, 4, p, f, p, 4, 256, 256, 2, 0, None) == -1              # f32 output
    assert lib.zl_fp8_block_gemm(ctypes.c_void_p(8), f, 4, p, f, p, 4, 256, 256, 0, 0, None) == -1   # misaligned


def test_layers_linear_checks_its_configuration(lib):
    from zhilight_b200 import _lib, layers
    with pytest.raises(_lib.ZLError):
        layers.Linear(200, 256, quant=10)                 # K % 128
    lin = layers.Linear(256, 256, quant=10)
    assert lin.quant == layers.QUANT_FP8_BLOCK
    with pytest.raises(_lib.ZLError):
        layers.Linear(256, 256, quant=9)


def _create(**kw):
    from zhilight_b200.llama import LlamaDecoder
    cfg = dict(num_layers=1, dim_model=256, num_heads=4, num_kv_heads=2, dim_head=64, dim_ff=512, vocab_size=512,
               eps=1e-5, rope_theta=10000.0, rope_llama3=None, quant_type=10, max_batch=2, max_seq=32)
    cfg.update(kw)
    return LlamaDecoder(**cfg)


@pytest.mark.parametrize("kw", [dict(tp_size=2), dict(qkv_bias=True), dict(dim_ff=576), dict(num_kv_heads=1),
                                dict(dim_model=320, num_heads=5)],
                         ids=["tp2", "qkv_bias", "ff%128", "kv%128", "D%128"])
def test_driver_refuses_unsupported_configurations(lib, kw):
    from zhilight_b200 import _lib
    with pytest.raises(_lib.ZLError) as e:
        _create(**kw)
    assert e.value.code == -2


def test_golden_from_reference_kernel_matches_oracle():
    """tests/golden/fp8_block_ref.npz holds the reference's own per_token_cast_to_fp8 outputs (codes and scales, f16 and
    bf16, column- and row-major scales, all-zero and clamped groups); the oracle reproduces them bit for bit."""
    from tests import fp8_block_golden as fg
    with np.load(fg.FIXTURE) as g:
        assert sorted(g.files) == sorted(k + s for _, _, _, k in fg.keys() for s in ("_q", "_s"))
        assert fg.check(g) == len(fg.keys())
