"""CPU tests of the oracle itself: internal consistency of the integer layout restatements, the float
restatements against independent formulas, and (when present) the golden vectors produced by the
reference's own kernels (tests/golden/ref_*.npz, see oracle/gen_ref_golden.py)."""
import glob
import os

import numpy as np
import pytest

from oracle import gptq, ops
from tests.helpers import rel_l2

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def test_shuffle_is_reference_nibble_order():
    # qdq_4.cuh:16-35 comment "77775555 33331111 66664444 22220000"
    w = np.array([0x76543210], dtype=np.uint32)
    out = gptq.shuffle_4bit_8(w)
    assert out[0] == 0x75316420


def test_k_major_roundtrip_matches_hf_unpack():
    k, n = 256, 64
    qw, qz, sc, gi = gptq.make_gptq_checkpoint(k, n, 128, False, seed=3)
    qw_km, qz_km, sc_km, perm = gptq.to_k_major(qw, qz, sc, gi, 128)
    assert perm is None
    assert qw_km.shape == (n, k // 8) and qz_km.shape == (n, 2) and sc_km.shape == (n, 2)
    q_nat = gptq.unpack_rows_u4(qw)                      # (K, N)
    np.testing.assert_array_equal(gptq.unpack_k_major(qw_km), q_nat.T)
    z_plus1 = (gptq.unpack_cols_u4(qz).astype(np.int32) + 1) & 15
    np.testing.assert_array_equal(qz_km, z_plus1.T.astype(np.uint8))
    w1 = gptq.dequant_k_major_f32(qw_km, qz_km, sc_km)
    w2 = gptq.hf_dequant_f32(qw, qz, sc, gi, 128)
    np.testing.assert_array_equal(w1, w2)


def test_increase_zero_wraps():
    w = np.array([0xFFFFFFFF, 0x00000000, 0x7E8F0123], dtype=np.uint32)
    out = gptq.increase_zero(w)
    assert list(out) == [0x00000000, 0x11111111, 0x8F901234]


def test_subtract8():
    w = np.array([0x0F87_1234], dtype=np.uint32)
    assert gptq.subtract8(w)[0] == 0x870F_9ABC


def test_act_order_gather():
    k, n, g = 256, 16, 128
    qw, qz, sc, _ = gptq.make_gptq_checkpoint(k, n, g, False, seed=5)
    rng = np.random.default_rng(0)
    g_idx = rng.permutation(np.arange(k) // g).astype(np.int32)
    perm = gptq.argsort_g_idx(g_idx, g)
    assert sorted(perm.tolist()) == list(range(k))
    assert np.all(g_idx[perm] == np.arange(k) // g)
    seq = gptq.make_sequential(qw, perm)
    np.testing.assert_array_equal(gptq.unpack_rows_u4(seq), gptq.unpack_rows_u4(qw)[perm])
    # act-order weights applied to permuted activations == original (linear.cpp:1010-1028, utils.cu:322-398)
    x = rng.standard_normal((2, k)).astype(np.float32)
    w_ref = gptq.hf_dequant_f32(qw, qz, sc, g_idx, g)
    qw_km, qz_km, sc_km, p2 = gptq.to_k_major(qw, qz, sc, g_idx, g)
    np.testing.assert_array_equal(p2, perm)
    w_perm = gptq.dequant_k_major_f32(qw_km, qz_km, sc_km)
    np.testing.assert_allclose(x[:, perm] @ w_perm.T, x @ w_ref.T, rtol=1e-5, atol=1e-4)


def test_awq_paths_agree():
    k, n, g = 128, 64, 128
    rng = np.random.default_rng(1)
    qw = rng.integers(0, 2 ** 32, size=(k, n // 8), dtype=np.uint64).astype(np.uint32)
    qz = rng.integers(0, 2 ** 32, size=(k // g, n // 8), dtype=np.uint64).astype(np.uint32)
    sc = (0.01 * rng.random((k // g, n))).astype(np.float16)
    q, z = gptq.awq_unpack(qw, qz)
    w_direct = ((q.astype(np.float32) - np.repeat(z.astype(np.float32), g, axis=0)) *
                np.repeat(sc.astype(np.float32), g, axis=0)).T
    qw_km, qz_km, sc_km, _ = gptq.to_k_major(qw, qz, sc, None, g, is_awq=True)
    np.testing.assert_array_equal(gptq.dequant_k_major_f32(qw_km, qz_km, sc_km), w_direct)
    # the non-exllama packing keeps natural k order inside a word
    nat = gptq.shuffle_awq(qw, use_exllama=False)
    np.testing.assert_array_equal(gptq.unpack_rows_u4(nat), q)


def test_reference_numerics_emulation_close_to_fp32():
    k, n = 256, 32
    qw, qz, sc, gi = gptq.make_gptq_checkpoint(k, n, 128, False, seed=7)
    qw_km, qz_km, sc_km, _ = gptq.to_k_major(qw, qz, sc, gi, 128)
    x = np.random.default_rng(2).standard_normal((2, k)).astype(np.float16)
    y32 = gptq.gemm_f32(x, gptq.dequant_k_major_f32(qw_km, qz_km, sc_km))
    yem = gptq.gemv_ref_numerics(x, qw_km, qz_km, sc_km).astype(np.float32)
    rel = np.linalg.norm(yem - y32) / np.linalg.norm(y32)
    assert rel < 3e-3


def test_dequant_f16_matches_f32_within_half_ulp():
    k, n = 128, 32
    qw, qz, sc, gi = gptq.make_gptq_checkpoint(k, n, 128, False, seed=8)
    qw_km, qz_km, sc_km, _ = gptq.to_k_major(qw, qz, sc, gi, 128)
    w16 = gptq.dequant_k_major_f16(qw_km, qz_km, sc_km).astype(np.float32)
    w32 = gptq.dequant_k_major_f32(qw_km, qz_km, sc_km)
    np.testing.assert_allclose(w16, w32, rtol=2 ** -10, atol=1e-6)


def test_rmsnorm_variants():
    rng = np.random.default_rng(3)
    a = rng.standard_normal((3, 64)).astype(np.float16)
    b = rng.standard_normal((3, 64)).astype(np.float16)
    w = (1 + 0.1 * rng.standard_normal(64)).astype(np.float16)
    h, y0 = ops.add_then_rmsnorm(a, b, w, 1e-5)
    s, y1 = ops.add_rmsnorm_fused(a, b, w, 1e-5)
    np.testing.assert_array_equal(h, s)
    np.testing.assert_allclose(y0, y1, rtol=2e-3, atol=2e-3)
    x = h
    ref = x / np.sqrt((x * x).mean(-1, keepdims=True) + 1e-5) * w.astype(np.float32)
    np.testing.assert_allclose(y0, ref, rtol=1e-3, atol=1e-3)


def test_rope_llama3_matches_hf_formula():
    d, theta = 64, 500000.0
    l3 = dict(factor=32.0, low=1.0, high=4.0, orig=8192.0)
    inv = ops.rope_inv_freq(d, theta, l3).astype(np.float64)
    base = 1.0 / (theta ** (np.arange(0, d, 2, dtype=np.float64) / d))
    wl = 2 * np.pi / base
    out = np.where(wl > 8192.0 / 1.0, base / 32.0, base)
    smooth = (8192.0 / wl - 1.0) / (4.0 - 1.0)
    mid = (1 - smooth) * out / 32.0 + smooth * out
    is_mid = ~(wl < 8192.0 / 4.0) & ~(wl > 8192.0 / 1.0)
    hf = np.where(is_mid, mid, out)
    np.testing.assert_allclose(inv, hf, rtol=1e-5)


def test_rope_neox_rotation_is_orthogonal():
    rng = np.random.default_rng(4)
    x = rng.standard_normal((5, 3, 64)).astype(np.float32)
    cos, sin = ops.rope_cos_sin(np.arange(5), 64, 10000.0)
    y = ops.rope_apply(x, cos, sin, True, "f32")
    np.testing.assert_allclose(np.linalg.norm(y, axis=-1), np.linalg.norm(x, axis=-1), rtol=1e-5)
    # position 0 is the identity
    np.testing.assert_allclose(y[0], x[0], atol=1e-6)


def test_decode_attention_against_plain_softmax():
    rng = np.random.default_rng(5)
    hq, hkv, d, lb = 4, 2, 16, 37
    q = rng.standard_normal((1, 1, hq, d)).astype(np.float16)
    k = rng.standard_normal((lb, hkv, d)).astype(np.float16)
    v = rng.standard_normal((lb, hkv, d)).astype(np.float16)
    mask = np.ones((1, lb), np.int8)
    mask[0, 30:] = 0
    o = ops.decode_attention(q, [k], [v], [lb], [mask], 0.25, 2, "f32")
    for h in range(hq):
        s = (k[:30, h // 2].astype(np.float64) @ q[0, 0, h].astype(np.float64)) * 0.25
        p = np.exp(s - s.max())
        p /= p.sum()
        np.testing.assert_allclose(o[0, 0, h], p @ v[:30, h // 2].astype(np.float64), rtol=1e-4, atol=1e-5)


def test_split_kv_combine_equals_full():
    rng = np.random.default_rng(6)
    s = rng.standard_normal(64).astype(np.float32)
    v = rng.standard_normal((64, 8)).astype(np.float32)
    full = (np.exp(s - s.max()) / np.exp(s - s.max()).sum()) @ v
    parts, ms, ls = [], [], []
    for a in range(0, 64, 16):
        ss = s[a:a + 16]
        e = np.exp(ss - ss.max())
        parts.append((e / e.sum()) @ v[a:a + 16])
        ms.append(ss.max())
        ls.append(e.sum())
    out = ops.split_kv_combine(np.stack(parts), np.array(ms), np.array(ls))
    np.testing.assert_allclose(out, full, rtol=1e-5, atol=1e-6)


def test_int8_allreduce_close_to_exact():
    rng = np.random.default_rng(7)
    for ws in (2, 4, 8):
        parts = [rng.standard_normal((4, 256)).astype(np.float16) for _ in range(ws)]
        q = ops.allreduce_int8_reference(parts)
        e = ops.allreduce_exact(parts)
        rel = np.linalg.norm(q - e) / np.linalg.norm(e)
        assert rel < 0.02, (ws, rel)


def test_int8_per_token_quant_roundtrip():
    rng = np.random.default_rng(8)
    x = rng.standard_normal((3, 128)).astype(np.float16)
    q, s = ops.int8_quant_per_token(x)
    assert np.abs(q).max() == 127
    np.testing.assert_allclose(q.astype(np.float32) * s[:, None], x.astype(np.float32), atol=float(s.max()) * 0.51)


def test_e4m3_rounding_grid():
    vals = np.array([0.0, 1.0, 1.0625, 1.125, 448.0, 500.0, -0.001953125, 2 ** -10], np.float32)
    out = ops.e4m3_round(vals)
    assert out[1] == 1.0 and out[3] == 1.125 and out[4] == 448.0 and out[5] == 448.0
    assert out[2] in (1.0, 1.125)            # tie -> even mantissa
    assert out[6] == -0.001953125            # 2^-9 is the smallest subnormal
    assert out[7] in (0.0, 0.001953125)


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "ref_*.npz"))) or [None])
def test_oracle_against_reference_goldens(path):
    """Goldens are outputs of the reference's own kernels (oracle/_ref, built from the reference checkout's sources)
    on seeded inputs; they pin the oracle.  Absent -> parity is 'unpinned' and this test is skipped."""
    if path is None:
        pytest.skip("no reference goldens committed yet (parity unpinned)")
    from oracle import check_golden
    check_golden.check_file(path)


def test_w8_oracle_functions_are_self_consistent():
    """INT8 / FP8 Linear restatements (oracle/ops.py): exact integer identities and closeness to the fp Linear."""
    rng = np.random.default_rng(21)
    x = ops._t(rng.standard_normal((6, 512)) * 1.3, "f16")
    w = ops._t(rng.standard_normal((96, 512)) * 0.05, "f16")
    wq, ws = ops.int8_weight_quant_per_row(w)
    q, s = ops.int8_quant_per_token(x)
    assert q.dtype == np.int8 and np.abs(q).max() == 127                    # every token reaches full scale
    np.testing.assert_allclose(q * s[:, None], x, atol=float(s.max()) * 0.5 + 1e-7)
    y = ops.int8_linear(x, wq, ops._t(ws, "f16"), "f16")
    assert rel_l2(y, x @ w.T) < 2e-2
    # all-zero token: quantises to zeros with scale 0 (device NaN -> int8 conversion), output row is exactly 0
    x0 = x.copy()
    x0[2] = 0
    q0, s0 = ops.int8_quant_per_token(x0)
    assert not q0[2].any() and s0[2] == 0
    # layernorm_quant: the int8 twin times its scale reproduces the normalised output
    ln_w = ops._t(1 + 0.1 * rng.standard_normal(512), "f16")
    yn, qn, sn = ops.rmsnorm_quant(x, ln_w, 1e-5, 1.0, "f16")
    np.testing.assert_allclose(qn * sn[:, None], yn, atol=float(sn.max()) * 0.51 + 2e-3)
    # e4m3: decode(encode) round trip on every finite code, saturation at 448
    codes = np.arange(256, dtype=np.uint8)
    vals = ops.e4m3_decode(codes)
    fin = np.isfinite(vals)
    np.testing.assert_array_equal(ops.e4m3_round(vals[fin]), vals[fin])
    assert ops.e4m3_round(np.array([1e6, -1e6], np.float32)).tolist() == [448.0, -448.0]
    xq, xs = ops.fp8_quant_per_tensor(x, dtype="f16")
    assert np.abs(xq).max() == 448.0
    y8 = ops.fp8_linear(x, ops.e4m3_round(w / 0.01), np.float32(0.01), "f16")
    assert rel_l2(y8, x @ w.T) < 6e-2


def test_w8_oracle_model_runs_and_tracks_the_fp_model():
    from oracle import model as omodel
    cfg = dict(num_layers=2, dim_model=256, num_heads=4, num_kv_heads=2, dim_head=64, dim_ff=512, vocab_size=512,
               eps=1e-5, rope_theta=10000.0, rope_llama3=None)
    sd = omodel.make_state_dict(cfg, 2, 128, False, seed=3)
    fp = omodel.OracleLlama(cfg, sd, 0, 128, False, "f16")
    i8 = omodel.OracleLlama(cfg, sd, 2, 128, False, "f16")
    tok = np.array([7, 300])
    a, b = fp.decode(tok, [0, 0]), i8.decode(tok, [0, 0])
    assert np.isfinite(b).all() and rel_l2(b, a) < 5e-2                      # SmoothQuant-level deviation
    sd8 = omodel.make_state_dict(cfg, 7, 128, False, seed=3)
    f8 = omodel.OracleLlama(cfg, sd8, 7, 128, False, "f16")
    assert np.isfinite(f8.decode(tok, [0, 0])).all()


def test_activation_digit_decomposition_identities():
    """The integer W4A16 kernel (zhilight_b200/csrc/w4a16_gemm_v3.cu) turns each 128-group of fp16 activations into
    integers m = round(x * 2^-e) and splits them into two 8-bit digits.  Restated here in numpy: both splittings are
    exact and the dot product with 4-bit weights reassembles exactly from the per-digit integer dot products."""
    rng = np.random.default_rng(5)
    x = (rng.standard_normal(128) * rng.choice([1e-3, 1.0, 300.0])).astype(np.float16).astype(np.float32)
    q = rng.integers(0, 16, size=128).astype(np.int64)
    for bits, packed in ((14, False), (13, True)):
        ex = int(np.frexp(np.abs(x).max())[1]) - 1 + 127          # biased exponent of the group maximum
        e = ex - 127 - bits
        m = np.rint(x * np.float32(2.0) ** -e).astype(np.int64)
        assert np.abs(m).max() <= 2 ** (bits + 1)
        if not packed:      # two IMMAs: signed high byte (floor), unsigned low byte
            hi, lo = m >> 8, m & 0xFF
            assert hi.min() >= -128 and hi.max() <= 127 and lo.min() >= 0
        else:               # one IMMA, both digits signed: lo' = int8(m & 0xff), hi' = (m + 128) >> 8
            lo = ((m & 0xFF) ^ 0x80) - 0x80
            hi = (m + 128) >> 8
            assert hi.min() >= -128 and hi.max() <= 127 and lo.min() >= -128 and lo.max() <= 127
        np.testing.assert_array_equal(hi * 256 + lo, m)
        # group dot product with the zero point removed through the exact sum of m (kernel epilogue)
        z = 8
        exact = int(((q - z) * m).sum())
        assert int((q * hi).sum()) * 256 + int((q * lo).sum()) - z * int(m.sum()) == exact
        # and the value it stands for is within 2^-(bits+1) of the group maximum of the fp32 product
        ref = float(((q - z) * x.astype(np.float64)).sum())
        tol = 128 * 15 * float(np.abs(x).max()) * 2.0 ** -(bits + 1)
        assert abs(exact * 2.0 ** e - ref) <= tol
