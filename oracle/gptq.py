"""CPU oracle: GPTQ / AWQ int4 layout transforms and W4A16 math (numpy).

TEST INFRASTRUCTURE -- see oracle/__init__.py.  Integer stages are bit-exact
restatements of the reference's load pipeline; float stages are fp32.

Reference files followed (paths inside the reference checkout):
  * nibble shuffle            src/nn/quant/gptq/qdq_4.cuh:16-35, q_gemm.cu:778-791
  * act-order gather          src/nn/quant/gptq/q_gemm.cu:794-829, linear.cpp:1010-1028
  * zero +1 with 4-bit wrap   src/nn/quant/gptq/utils.cu:61-88
  * q4 -> q8                  src/nn/quant/gptq/utils.cu:177-214
  * order of load-time ops    src/nn/linear/linear.cpp:1085-1099, 1139-1160
  * AWQ de-interleave         src/nn/quant/gptq/utils.cu:25-58, 121-174
  * dequant formula/numerics  src/nn/quant/gptq/q_gemm_k_major.cu:52-118, 127-173, 843-905
"""
import numpy as np

U32 = np.uint32


# ----------------------------------------------------------------------------
# HF-checkpoint (AutoGPTQ v1) tensor helpers -- linear.cpp:683-686
# ----------------------------------------------------------------------------
def unpack_rows_u4(qweight_k8_n):
    """(K/8, N) int32/uint32 -> (K, N) uint8; q[k,n] = (w[k>>3,n] >> 4*(k&7)) & 15."""
    w = np.ascontiguousarray(qweight_k8_n).view(U32)
    k8, n = w.shape
    out = np.empty((k8, 8, n), dtype=np.uint8)
    for i in range(8):
        out[:, i, :] = (w >> U32(4 * i)) & U32(0xF)
    return out.reshape(k8 * 8, n)


def unpack_cols_u4(qzeros_g_n8):
    """(G, N/8) int32 -> (G, N) uint8; z[g,n] = (w[g,n>>3] >> 4*(n&7)) & 15."""
    w = np.ascontiguousarray(qzeros_g_n8).view(U32)
    g, n8 = w.shape
    out = np.empty((g, n8, 8), dtype=np.uint8)
    for i in range(8):
        out[:, :, i] = (w >> U32(4 * i)) & U32(0xF)
    return out.reshape(g, n8 * 8)


def pack_rows_u4(q_k_n):
    """Inverse of unpack_rows_u4: (K, N) uint8 -> (K/8, N) uint32."""
    k, n = q_k_n.shape
    q = q_k_n.reshape(k // 8, 8, n).astype(U32)
    w = np.zeros((k // 8, n), dtype=U32)
    for i in range(8):
        w |= q[:, i, :] << U32(4 * i)
    return w


def pack_cols_u4(z_g_n):
    """Inverse of unpack_cols_u4: (G, N) uint8 -> (G, N/8) uint32."""
    g, n = z_g_n.shape
    z = z_g_n.reshape(g, n // 8, 8).astype(U32)
    w = np.zeros((g, n // 8), dtype=U32)
    for i in range(8):
        w |= z[:, :, i] << U32(4 * i)
    return w


# ----------------------------------------------------------------------------
# Load-time integer transforms (bit-exact targets)
# ----------------------------------------------------------------------------
def shuffle_4bit_8(words):
    """qdq_4.cuh:16-35.  nibbles [q0..q7] -> bits 0-15 = [q0,q2,q4,q6], bits 16-31 = [q1,q3,q5,q7]."""
    qa = np.ascontiguousarray(words).view(U32).copy()
    qb = np.zeros_like(qa)
    for i in range(4):
        qa0 = qa & U32(0x0F)
        qa1 = (qa & U32(0xF0)) >> U32(4)
        qa = qa >> U32(8)
        qb |= qa1 << U32(i * 4 + 16)
        qb |= qa0 << U32(i * 4)
    return qb


def argsort_g_idx(g_idx, group_size):
    """linear.cpp:1010-1028 (argsort_cpu): stable bucket sort of k by group id."""
    g_idx = np.asarray(g_idx, dtype=np.int64)
    numel = g_idx.size
    idx = np.zeros(numel, dtype=np.int32)
    count = np.zeros(numel // group_size, dtype=np.int64)
    for i in range(numel):
        x = g_idx[i]
        y = x * group_size + count[x]
        count[x] += 1
        assert y <= numel and count[x] <= group_size
        idx[y] = i
    return idx


def make_sequential(qweight_k8_n, q_perm):
    """q_gemm.cu:794-829: new row r of the (K, N) nibble matrix = old row q_perm[r]."""
    q = unpack_rows_u4(qweight_k8_n)
    return pack_rows_u4(q[np.asarray(q_perm, dtype=np.int64), :])


def gptq_shuffle(qweight_k8_n, q_perm=None):
    """q_gemm.cu:831-872 (shuffle_exllama_weight): optional act-order gather then shuffle_4bit_8."""
    w = np.ascontiguousarray(qweight_k8_n).view(U32)
    if q_perm is not None and len(q_perm):
        w = make_sequential(w, q_perm)
    return shuffle_4bit_8(w)


def increase_zero(qzeros):
    """utils.cu:61-88: every 4-bit field z := (z + 1) & 0xF (15 wraps to 0)."""
    w = np.ascontiguousarray(qzeros).view(U32)
    out = np.zeros_like(w)
    for i in range(8):
        nib = (w >> U32(4 * i)) & U32(0xF)
        out |= ((nib + U32(1)) & U32(0xF)) << U32(4 * i)
    return out


def subtract8(words):
    """utils.cu:91-118: every 4-bit field q := (q >= 8) ? q - 8 : q + 8  (i.e. q ^ 8)."""
    w = np.ascontiguousarray(words).view(U32)
    return w ^ U32(0x88888888)


def q4_to_q8(qzeros_g_n8):
    """utils.cu:177-214: (G, N/8) int32 -> (G, N) uint8, nibble j of a word -> byte j."""
    return unpack_cols_u4(qzeros_g_n8)


def q8_to_q4(z_g_n):
    """utils.cu:217-250 inverse of q4_to_q8."""
    return pack_cols_u4(z_g_n)


AWQ_DE_SFL = (0, 4, 1, 5, 2, 6, 3, 7)   # utils.cu:33,132
EXL_SFL = (0, 2, 4, 6, 1, 3, 5, 7)      # utils.cu:147


def un_shuffle(qzeros):
    """utils.cu:25-58: out nibble s = in nibble de_sfl[s] (AWQ column de-interleave)."""
    w = np.ascontiguousarray(qzeros).view(U32)
    out = np.zeros_like(w)
    for s in range(8):
        out |= ((w >> U32(AWQ_DE_SFL[s] * 4)) & U32(0xF)) << U32(s * 4)
    return out


def shuffle_awq(qweight_k_n8, use_exllama=True):
    """utils.cu:121-174: AWQ (K, N/8) -> GPTQ (K/8, N); de-interleave columns, then pack 8
    consecutive k per word in exllama order [0,2,4,6,1,3,5,7] (or natural order)."""
    w = np.ascontiguousarray(qweight_k_n8).view(U32)
    k, n8 = w.shape
    dq = np.empty((k, n8, 8), dtype=U32)          # dq[k, n8, c] = logical column 8*n8 + c
    for s in range(8):
        dq[:, :, s] = (w >> U32(AWQ_DE_SFL[s] * 4)) & U32(0xF)
    dq = dq.reshape(k // 8, 8, n8 * 8)            # [k8, r, n]
    out = np.zeros((k // 8, n8 * 8), dtype=U32)
    for s in range(8):
        r = EXL_SFL[s] if use_exllama else s
        out |= dq[:, r, :] << U32(s * 4)
    return out


def awq_unpack(qweight_k_n8, qzeros_g_n8):
    """AWQ logical nibbles: q (K, N), z (G, N) uint8 (awq/dequantize.cuh:45-112 ordering)."""
    def unp(w):
        w = np.ascontiguousarray(w).view(U32)
        r, c8 = w.shape
        o = np.empty((r, c8, 8), dtype=np.uint8)
        for s in range(8):
            o[:, :, s] = (w >> U32(AWQ_DE_SFL[s] * 4)) & U32(0xF)
        return o.reshape(r, c8 * 8)
    return unp(qweight_k_n8), unp(qzeros_g_n8)


def to_k_major(qweight, qzeros, scales, g_idx=None, group_size=128, is_awq=False):
    """Full reference load pipeline (linear.cpp:1139-1160 preprocess_weight + 1085-1099
    transpose_weight) for the default kernel (GPTQ_KERNEL_ALGO=1, use_exllama=True).

    Returns (qweight_km (N,K/8) uint32, qzeros_km (N,G) uint8, scales_km (N,G) float16, q_perm)
    where q_perm is the act-order permutation (argsort of g_idx) or None.
    """
    q_perm = None
    if is_awq:
        qw = shuffle_awq(qweight, True)
        qz = un_shuffle(qzeros)
    else:
        if g_idx is not None:
            g_idx = np.asarray(g_idx)
            k = g_idx.size
            if not np.array_equal(g_idx, np.arange(k) // group_size):
                q_perm = argsort_g_idx(g_idx, group_size)
        qw = gptq_shuffle(qweight, q_perm)
        qz = increase_zero(qzeros)
    z8 = q4_to_q8(qz)                                   # (G, N) u8
    return (np.ascontiguousarray(qw.T), np.ascontiguousarray(z8.T),
            np.ascontiguousarray(np.asarray(scales, dtype=np.float16).T), q_perm)


# ----------------------------------------------------------------------------
# k-major decode + math
# ----------------------------------------------------------------------------
def unpack_k_major(qweight_km):
    """(N, K/8) shuffled words -> (N, K) uint8 in natural k order
    (q_gemm_k_major.cu:74-98: masks 0x000f000f / 0x00f000f0, then >> 8)."""
    w = np.ascontiguousarray(qweight_km).view(U32)
    n, k8 = w.shape
    out = np.empty((n, k8, 8), dtype=np.uint8)
    for i in range(4):
        out[:, :, 2 * i] = (w >> U32(4 * i)) & U32(0xF)
        out[:, :, 2 * i + 1] = (w >> U32(4 * i + 16)) & U32(0xF)
    return out.reshape(n, k8 * 8)


def dequant_k_major_f32(qweight_km, qzeros_km, scales_km, sym=False):
    """W[n,k] = (q[n,k] - z[n,k/g]) * s[n,k/g] in fp32.  sym -> z == 8
    (q_gemm_k_major.cu:148-150)."""
    q = unpack_k_major(qweight_km).astype(np.float32)
    n, k = q.shape
    g = scales_km.shape[1]
    gs = k // g
    z = np.full((n, g), 8.0, np.float32) if sym else np.asarray(qzeros_km).astype(np.float32)
    s = np.asarray(scales_km).astype(np.float32)
    return (q - np.repeat(z, gs, axis=1)) * np.repeat(s, gs, axis=1)


def dequant_k_major_f16(qweight_km, qzeros_km, scales_km):
    """KERNEL_dequant OUT_TYPE=0 (q_gemm_k_major.cu:843-881): half(q - z) * half(s) rounded to
    fp16; always uses the stored zeros."""
    q = unpack_k_major(qweight_km).astype(np.float16)
    n, k = q.shape
    g = scales_km.shape[1]
    gs = k // g
    z = np.asarray(qzeros_km).astype(np.float16)
    s = np.asarray(scales_km).astype(np.float16)
    return ((q - np.repeat(z, gs, axis=1)) * np.repeat(s, gs, axis=1)).astype(np.float16)


def gemm_f32(x, w_f32, bias=None):
    """y = x @ W^T (+ bias) in fp32; x (M,K) any float dtype, W (N,K)."""
    y = np.asarray(x).astype(np.float32) @ np.asarray(w_f32, dtype=np.float32).T
    if bias is not None:
        y = y + np.asarray(bias).astype(np.float32)[None, :]
    return y


def gemv_ref_numerics(x, qweight_km, qzeros_km, scales_km, sym=False, bias=None):
    """Emulates KERNEL_gemm_warp_reduce numerics (q_gemm_k_major.cu:101-108,127-237):
    per packed word the 8 products are accumulated in fp16 as two 4-step fma chains
    (lanes k even / k odd), widened, summed, scaled in fp32; lane l owns words l, l+32, ...
    accumulated sequentially in fp32; shfl_down tree; output cast to fp16.
    Small sizes only (python loops over words)."""
    x = np.asarray(x).astype(np.float16)
    m, k = x.shape
    q = unpack_k_major(qweight_km).astype(np.float32)          # (N, K)
    n = q.shape[0]
    g = scales_km.shape[1]
    gs = k // g
    z = np.full((n, g), 8.0, np.float32) if sym else np.asarray(qzeros_km).astype(np.float32)
    dq = (q - np.repeat(z, gs, axis=1)).astype(np.float16)     # exact small ints
    s = np.asarray(scales_km).astype(np.float32)
    k8 = k // 8
    out = np.zeros((m, n), dtype=np.float16)
    for mi in range(m):
        xa = x[mi].reshape(k8, 8)
        lane_acc = np.zeros((32, n), dtype=np.float32)
        for w in range(k8):
            d = dq[:, w * 8:(w + 1) * 8]                        # (N, 8) fp16
            lo = np.zeros(n, dtype=np.float16)
            hi = np.zeros(n, dtype=np.float16)
            for i in range(4):
                # __hfma2: single rounding of d*a + acc to fp16
                lo = (d[:, 2 * i].astype(np.float32) * np.float32(xa[w, 2 * i]) + lo.astype(np.float32)).astype(np.float16)
                hi = (d[:, 2 * i + 1].astype(np.float32) * np.float32(xa[w, 2 * i + 1]) + hi.astype(np.float32)).astype(np.float16)
            dot = lo.astype(np.float32) + hi.astype(np.float32)
            sc = s[:, (w * 8) // gs]
            lane = w % 32
            # fma(dot, scale, acc) -- single rounding, emulate in float64 then round
            lane_acc[lane] = (dot.astype(np.float64) * sc.astype(np.float64) + lane_acc[lane].astype(np.float64)).astype(np.float32)
        v = lane_acc.copy()
        off = 16
        while off > 0:
            nv = v.copy()
            nv[:32 - off] = v[:32 - off] + v[off:]
            v = nv
            off //= 2
        acc = v[0]
        if bias is not None:
            acc = acc + np.asarray(bias).astype(np.float32)
        out[mi] = acc.astype(np.float16)
    return out


# ----------------------------------------------------------------------------
# Synthetic checkpoints (SURVEY.md section 8d config 1 / 3 generators)
# ----------------------------------------------------------------------------
def make_gptq_checkpoint(k, n, group_size=128, sym=False, seed=0, scale_lo=0.005, scale_hi=0.02):
    """HF-GPTQ tensors with uniform random nibbles.  sym=True stores zeros == 7 (-> 8 after +1)."""
    rng = np.random.default_rng(seed)
    qweight = rng.integers(0, 2 ** 32, size=(k // 8, n), dtype=np.uint64).astype(U32)
    if sym:
        qzeros = np.full((k // group_size, n // 8), 0x77777777, dtype=U32)
    else:
        qzeros = rng.integers(0, 2 ** 32, size=(k // group_size, n // 8), dtype=np.uint64).astype(U32)
    scales = (scale_lo + (scale_hi - scale_lo) * rng.random((k // group_size, n))).astype(np.float16)
    g_idx = (np.arange(k) // group_size).astype(np.int32)
    return qweight.view(np.int32), qzeros.view(np.int32), scales, g_idx


def hf_dequant_f32(qweight, qzeros, scales, g_idx=None, group_size=128):
    """Straight-from-checkpoint dequant, reference semantics (wrapped +1 zero):
    W[k,n] = (q[k,n] - ((z[g(k),n] + 1) & 15)) * s[g(k),n]  ->  returns (N, K) fp32."""
    q = unpack_rows_u4(qweight).astype(np.float32)                 # (K, N)
    z = ((unpack_cols_u4(qzeros).astype(np.int32) + 1) & 15).astype(np.float32)   # (G, N)
    s = np.asarray(scales).astype(np.float32)
    k = q.shape[0]
    gi = np.arange(k) // group_size if g_idx is None else np.asarray(g_idx)
    w = (q - z[gi, :]) * s[gi, :]
    return np.ascontiguousarray(w.T)
