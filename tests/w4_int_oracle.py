"""Float64 restatement of the exact-integer W4A16 kernel's arithmetic (k_w4a16_v3, zhilight_b200/csrc/w4a16_gemm_v3.cu),
with an elementwise bound of its distance to the exact GEMM of the unquantised activations.

Per token and 128-group the kernel stages  x' = fp16(x * ln_w)  (x alone without the fused RMSNorm; x[k_perm] and
ln_w[k_perm] with act-order), takes the block exponent  e = floor(log2 max|x'|) - kE  (kE = 14, 13 for the digit-packed
PACK variants) and the integer mantissas  m = rint(x' * 2^-e).  A group whose fp32 exponent field is below 20 is all-zero;
a non-finite group poisons its token with NaN.  r_g = sum (q - z) * m  is exact (int32 IMMA), and
y = fp16(rstd * sum_g r_g * s_g * 2^e_g + bias), then the RESIDUAL, SWIGLU or QKV_ROPE epilogue.

Weights here are in PACKED row order (the order the kernel's tiles and bias use): q (N, K) nibbles, z (N, G), s (N, G).
"""
import numpy as np

GROUP = 128
KE, KE_PACK = 14, 13
F32_EPS = 2.0 ** -24


def pack_k_major(q):
    """(N, K) nibbles -> (N, K/8) uint32 k-major words: the inverse of oracle.gptq.unpack_k_major (k 2i at bits 4i, k 2i+1
    at bits 4i + 16)."""
    q = np.asarray(q, dtype=np.uint32)
    n, k = q.shape
    q = q.reshape(n, k // 8, 8)
    w = np.zeros((n, k // 8), dtype=np.uint32)
    for i in range(4):
        w |= q[:, :, 2 * i] << np.uint32(4 * i)
        w |= q[:, :, 2 * i + 1] << np.uint32(4 * i + 16)
    return w


def f16(a):
    return np.asarray(a, dtype=np.float64).astype(np.float16).astype(np.float64)


def ulp16(a):
    """one fp16 ulp at magnitude |a| (2^-24 in the subnormal range)"""
    a = np.abs(np.asarray(a, dtype=np.float64))
    _, p = np.frexp(np.maximum(a, 2.0 ** -14))
    return np.ldexp(1.0, p - 11)


def stage(x, ln_w=None, k_perm=None):
    """the fp16 values the kernel quantises (M, K) and the un-multiplied x the RMS is taken over"""
    x = np.asarray(x, dtype=np.float16)
    if k_perm is not None:
        x = x[:, k_perm]
    if ln_w is None:
        return x.astype(np.float64), x.astype(np.float64)
    lw = np.asarray(ln_w, dtype=np.float16)
    if k_perm is not None:
        lw = lw[k_perm]
    with np.errstate(over="ignore", invalid="ignore"):
        xn = (x.astype(np.float32) * lw.astype(np.float32)).astype(np.float16)   # __hmul2: one rounding of an exact product
    return xn.astype(np.float64), x.astype(np.float64)


def quantise(xs, pack, ke=None, drop_group=None):
    """block-floating-point decomposition of the staged activations: m (M, K) float64 integers, e (M, G) exponents,
    live (M, G) (group neither all-zero nor poisoned), poison (M) bool.  ke / drop_group exist to break the oracle on
    purpose in its own tests."""
    ke = (KE_PACK if pack else KE) if ke is None else ke
    m_, k = xs.shape
    g = k // GROUP
    xg = xs.reshape(m_, g, GROUP)
    with np.errstate(invalid="ignore"):
        amax = np.max(np.abs(xg), axis=2)
    finite = np.isfinite(amax)
    live = finite & (amax >= 2.0 ** (20 - 127))            # fp32 exponent field >= 20
    _, p = np.frexp(np.where(live, amax, 1.0))
    e = np.where(live, p - 1 - ke, 0)
    with np.errstate(invalid="ignore"):
        m = np.rint(np.ldexp(np.where(live[:, :, None], xg, 0.0), -e[:, :, None]))
    if drop_group is not None:
        live = live.copy()
        live[:, drop_group] = False
    m = np.where(live[:, :, None], m, 0.0)
    return m.reshape(m_, k), e, live, ~finite.all(axis=1)


def gemm(x, q, z, s, *, pack, ln_w=None, eps=1e-5, k_perm=None, bias=None, ke=None, drop_group=None):
    """Pre-epilogue values of every (token, packed row), transposed to (M, N):
      v      the kernel's arithmetic in float64 (before its final fp16 rounding)
      exact  rstd * W . x' + bias in float64: the exact GEMM of the unquantised staged activations
      qb     the bound of |v - exact|: rstd * sum_g |s_g| sum_k |q - z| 2^(e_g - 1)
      f32    the bound of the kernel's fp32 rounding (int -> float, one fma per group, the split-k sum, rstd, bias)
      poison (M) tokens the kernel sets to NaN"""
    q = np.asarray(q)
    n, k = q.shape
    g = k // GROUP
    xs, xraw = stage(x, ln_w, k_perm)
    m, e, live, poison = quantise(xs, pack, ke, drop_group)
    mt = xs.shape[0]
    if ln_w is not None:
        with np.errstate(over="ignore", invalid="ignore"):
            rstd = 1.0 / np.sqrt(np.sum(xraw * xraw, axis=1) / k + eps)
    else:
        rstd = np.ones(mt)
    rstd = np.where(np.isfinite(rstd), rstd, 0.0)
    zf = np.asarray(z, dtype=np.float64)
    sf = np.asarray(s, dtype=np.float16).astype(np.float64)
    v = np.zeros((n, mt))
    a = np.zeros((n, mt))
    qb = np.zeros((n, mt))
    ex = np.zeros((n, mt))
    xe = np.where(np.isfinite(xs), xs, 0.0)
    for gi in range(g):
        d = q[:, gi * GROUP:(gi + 1) * GROUP].astype(np.float64) - zf[:, gi:gi + 1]      # q - z, exact
        r = d @ m[:, gi * GROUP:(gi + 1) * GROUP].T                                       # exact: |r| < 2^31
        scale = sf[:, gi:gi + 1] * np.ldexp(1.0, e[:, gi])[None, :]
        term = r * scale
        v += term
        a += np.abs(term)
        half = np.where(live[:, gi], np.ldexp(1.0, e[:, gi] - 1), 0.0)
        # a group the kernel skips as all-zero holds values below 2^-107: their whole magnitude is the error
        lost = np.where(live[:, gi], 0.0, np.max(np.abs(xe[:, gi * GROUP:(gi + 1) * GROUP]), axis=1))
        qb += (np.abs(d).sum(axis=1, keepdims=True) * np.abs(sf[:, gi:gi + 1])) * (half + lost)[None, :]
        ex += (d * sf[:, gi:gi + 1]) @ xe[:, gi * GROUP:(gi + 1) * GROUP].T
    b = np.zeros(n) if bias is None else np.asarray(bias, dtype=np.float16).astype(np.float64)
    v = (v * rstd[None, :]).T + b[None, :]
    ex = (ex * rstd[None, :]).T + b[None, :]
    a = (a * rstd[None, :]).T + np.abs(b)[None, :]
    qb = (qb * rstd[None, :]).T
    f32 = (2 * g + 96) * F32_EPS * a
    return dict(v=v, exact=ex, qb=qb, f32=f32, poison=poison)


# ---- epilogues: (value, tolerance) of each output element given pre-epilogue values v within dv of the kernel's ----
def epi_none(v, dv):
    return v, dv + ulp16(np.abs(v) + dv)


def epi_residual(v, dv, res):
    res = np.asarray(res, dtype=np.float16).astype(np.float64)
    d1 = dv + ulp16(np.abs(v) + dv)                          # h = fp16(v)
    out = v + res
    return out, d1 + ulp16(np.abs(out) + d1)                 # fp16(h + residual)


def _silu(x):
    return x / (1.0 + np.exp(-x))


def epi_swiglu(v, dv):
    """y[:, t * 16 + oc] = fp16(silu(fp16(gate)) * fp16(up)), gate / up = packed rows t*32 + rg, rg + 8 with
    rg = (oc >> 3) * 16 + (oc & 7)"""
    mt, n = v.shape
    oc = np.arange(n // 2) % 16
    rg = (np.arange(n // 2) // 16) * 32 + (oc >> 3) * 16 + (oc & 7)
    g, u, dg, du = v[:, rg], v[:, rg + 8], dv[:, rg], dv[:, rg + 8]
    dg = dg + ulp16(np.abs(g) + dg)
    du = du + ulp16(np.abs(u) + du)
    with np.errstate(over="ignore"):
        sg = _silu(g)
    out = sg * u
    tol = 1.1 * (np.abs(u) + du) * dg + (np.abs(sg) + 1.1 * dg) * du + 2.0 ** -20 * (np.abs(sg) + 1.1 * dg) * (np.abs(u) + du)
    return out, tol + ulp16(np.abs(out) + tol)


def epi_qkv(v, dv, cos, sin, hq, hkv, d):
    """(q (M, hq, d), k (M, hkv, d), v (M, hkv, d)) values and tolerances: tile st of head st / (d/32) holds, for oc < 16,
    columns c = jt*16 + oc (packed row rlo = (oc>>3)*16 + (oc&7)) and c + d/2 (row rlo + 8); q and k heads are rotated with
    the fp32 cos / sin tables, v heads are stored as they are"""
    mt, n = v.shape
    tiles = d // 32
    half = d // 2
    out = np.zeros((mt, hq + 2 * hkv, d))
    tol = np.zeros_like(out)
    cos = np.asarray(cos, dtype=np.float64)
    sin = np.asarray(sin, dtype=np.float64)
    for st in range(n // 32):
        head, jt = st // tiles, st % tiles
        for oc in range(16):
            rlo = st * 32 + (oc >> 3) * 16 + (oc & 7)
            c = jt * 16 + oc
            lo, hi = v[:, rlo], v[:, rlo + 8]
            dlo = dv[:, rlo] + ulp16(np.abs(v[:, rlo]) + dv[:, rlo])
            dhi = dv[:, rlo + 8] + ulp16(np.abs(v[:, rlo + 8]) + dv[:, rlo + 8])
            if head >= hq + hkv:
                olo, ohi, tlo, thi = lo, hi, dlo, dhi
            else:
                cl, sl, ch, sh = cos[:, c], sin[:, c], cos[:, c + half], sin[:, c + half]
                olo = lo * cl - hi * sl
                ohi = hi * ch + lo * sh
                tlo = np.abs(cl) * dlo + np.abs(sl) * dhi + 4 * F32_EPS * (np.abs(lo * cl) + np.abs(hi * sl) + dlo + dhi)
                thi = np.abs(ch) * dhi + np.abs(sh) * dlo + 4 * F32_EPS * (np.abs(hi * ch) + np.abs(lo * sh) + dlo + dhi)
            out[:, head, c], out[:, head, c + half] = olo, ohi
            tol[:, head, c] = tlo + ulp16(np.abs(olo) + tlo)
            tol[:, head, c + half] = thi + ulp16(np.abs(ohi) + thi)
    return out, tol


def epilogue(kind, v, dv, **kw):
    if kind == "none":
        return epi_none(v, dv)
    if kind == "res":
        return epi_residual(v, dv, kw["residual"])
    if kind == "swiglu":
        return epi_swiglu(v, dv)
    return epi_qkv(v, dv, kw["cos"], kw["sin"], kw["hq"], kw["hkv"], kw["d"])
