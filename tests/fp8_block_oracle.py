"""CPU oracle of the FP8 block-scaled Linear (QuantType 10, Fp8Block, src/nn/linear/linear.cpp:1697-1960).

quant_per_token_group restates nn::fp8::per_token_cast_to_fp8 (src/nn/quant/fp8/fp8_util.cu:231-322) exactly:
amax per (token, 128-column group) clamped to 1e-4, q = e4m3(satfinite(x * float32(448/amax))) with the fp32
product, scale = float32(amax/448) stored column-major (K/128, round_up(M, 4)).  block_gemm sums the decoded codes of
each 128-k block in float64 and applies x_scale[kb, m] * w_scale[n/128, kb] per block.
"""
import numpy as np

from oracle import ops

F32 = np.float32
_POS = ops.e4m3_decode(np.arange(0x7F, dtype=np.uint8)).astype(np.float64)   # codes 0x00 .. 0x7e, ascending


def e4m3_encode(v):
    """fp32 values -> e4m3fn bytes with RNE and saturation to +-448 (cvt.rn.satfinite.e4m3): the sign bit follows
    the input's, so a negative value that rounds to zero is 0x80 as on the GPU."""
    v = np.asarray(v, F32)
    r = np.abs(ops.e4m3_round(v).astype(np.float64))
    code = np.searchsorted(_POS, r).astype(np.uint8)
    return np.where(np.signbit(v), code | np.uint8(0x80), code).astype(np.uint8)


def scale_ld(m):
    return (m + 3) // 4 * 4


def quant_per_token_group(x):
    """x (M, K) values of f16/bf16 (as fp32) -> (codes uint8 (M, K), scales f32 (K/128, round_up(M, 4)))."""
    x = np.asarray(x, F32)
    m, k = x.shape
    assert k % 128 == 0
    g = x.reshape(m, k // 128, 128)
    amax = np.abs(g).max(axis=2).astype(F32)
    amax = np.where(amax < F32(1e-4), F32(1e-4), amax).astype(F32)
    mul = (F32(448.0) / amax).astype(F32)
    prod = (g * mul[:, :, None]).astype(F32)
    codes = e4m3_encode(prod).reshape(m, k)
    sc = np.zeros((k // 128, scale_ld(m)), F32)
    sc[:, :m] = (amax / F32(448.0)).astype(F32).T
    return codes, sc


def block_gemm(xq, x_scale, wq, w_scale, w_values=None):
    """y[m, n] = sum_kb (sum_{k in kb} x[m, k] w[n, k]) * x_scale[kb, m] * w_scale[n // 128, kb], in float64.
    xq (M, K) and wq (N, K) are e4m3 bytes.  w_values: the decoded weight (N, K) as float32 instead of wq, for models
    (a block's 128 products of e4m3 values then sum in fp32, exact to ~1e-7)."""
    xv = ops.e4m3_decode(xq).astype(np.float64)
    if w_values is None:
        wv = ops.e4m3_decode(wq).astype(np.float64)
    else:
        wv, xv = w_values, xv.astype(F32)
    m, k = xv.shape
    n = wv.shape[0]
    kb_n = k // 128
    sx = np.asarray(x_scale, np.float64)[:kb_n, :m]                     # (KB, M)
    sw = np.asarray(w_scale, np.float64)[np.arange(n) // 128]           # (N, KB)
    y = np.zeros((m, n))
    for kb in range(kb_n):
        part = (xv[:, kb * 128:(kb + 1) * 128] @ wv[:, kb * 128:(kb + 1) * 128].T).astype(np.float64)
        y += part * sx[kb][:, None] * sw[:, kb][None, :]
    return y


def linear(x, wq, w_scale, w_values=None):
    """Fp8Block::forward: quantise x per token group, then the block-scaled GEMM (float64, before the output cast)."""
    q, s = quant_per_token_group(x)
    return block_gemm(q, s, wq, w_scale, w_values)


def random_weight(n, k, rng, lo=1e-3, hi=1e2):
    """e4m3 weight codes (N, K) with the exponent MSB cleared (|w| < 2, no NaN codes, so fp16 outputs stay finite) and
    block scales (ceil(N/128), K/128) drawn log-uniformly over [lo, hi] so that a wrong block index or a scale applied
    after the k-sum shows."""
    codes = rng.integers(0, 256, size=(n, k), dtype=np.uint8) & np.uint8(0xBF)
    sw = np.exp(rng.uniform(np.log(lo), np.log(hi), size=((n + 127) // 128, k // 128))).astype(F32)
    return codes, sw


def dequant_weight(wq, w_scale):
    """nn::fp8::dequant_fp8_block_weight (fp8_util.cu:322-385): float(code) * scale[n/128, k/128] in fp32."""
    wv = ops.e4m3_decode(wq)
    n, k = wv.shape
    s = np.asarray(w_scale, F32)[np.arange(n) // 128][:, np.arange(k) // 128]
    return (wv * s).astype(F32)
