"""CPU oracle: RMSNorm / residual / RoPE / SwiGLU / decode attention / INT8 / FP8 /
int8 TP all-reduce (numpy, fp32 math).

TEST INFRASTRUCTURE -- see oracle/__init__.py.

Reference files followed (paths inside the reference checkout):
  * RMSNorm (+fused add)      src/nn/layernorm/layernorm.cu:9-42
  * residual add              src/nn/block/block_kernel.cu:7-17
  * RoPE                      src/nn/position/rope_common.cuh:3-34, rope_preparer.cu:49-161,
                              rotary_embedding_fuse_cache.cu:23-63
  * SiLU / gate mul           src/nn/functions/activation.cuh:8-14, linear/activation_kernel.cu:71-80
  * decode attention          src/nn/attention/attention_kernel.cu:434-489 (softmax),
                              674-725 (mqa_rag_buffer1), 730-923 (split-kv + combine)
  * KV append                 src/kvcache/ragged_buffer_kernel.cu:194-222
  * INT8 act quant / dequant  src/nn/quant/int8/quant_kernel.cu:15-47, 231-246
  * FP8 per-tensor quant      src/nn/quant/fp8/fp8_util.cu:58-147, 176-228
  * int8 TP all-reduce        src/nn/quant/int8/quant_reduce_kernel.cu:14-38, 105-140, 201-274,
                              src/model/model_context.cpp:244-326
"""
import math
import numpy as np

F32 = np.float32


def _t(x, dtype):
    """Round to the activation dtype T ('f16' or 'bf16') and come back as float32 values."""
    x = np.asarray(x, dtype=F32)
    if dtype in ("f16", "half", np.float16):
        return x.astype(np.float16).astype(F32)
    if dtype in ("bf16",):
        u = x.view(np.uint32).astype(np.uint64)
        # round to nearest even on the upper 16 bits
        r = ((u >> 16) & 1) + 0x7FFF
        u = ((u + r) >> 16) << 16
        return u.astype(np.uint32).view(F32)
    if dtype in ("f32", np.float32):
        return x
    raise ValueError(dtype)


# ----------------------------------------------------------------------------
# RMSNorm / residual
# ----------------------------------------------------------------------------
def rmsnorm(x, weight, eps, scale=1.0, dtype="f16"):
    """layernorm.cu:9-42 without add: y = T(x * rsqrt(mean(x^2)+eps) * w / scale)."""
    x = np.asarray(x, dtype=F32)
    w = np.asarray(weight, dtype=F32)
    ms = (x * x).sum(-1, keepdims=True, dtype=F32) / F32(x.shape[-1])
    r = F32(1.0) / np.sqrt(ms + F32(eps))
    return _t(x * r * w / F32(scale), dtype)


def add_rmsnorm_fused(a, b, weight, eps, scale=1.0, dtype="f16"):
    """layernorm.cu:28-41 fused-add variant: out_sum = T(a+b); norm uses the UNROUNDED fp32 sum."""
    v = np.asarray(a, dtype=F32) + np.asarray(b, dtype=F32)
    out_sum = _t(v, dtype)
    ms = (v * v).sum(-1, keepdims=True, dtype=F32) / F32(v.shape[-1])
    r = F32(1.0) / np.sqrt(ms + F32(eps))
    return out_sum, _t(v * r * np.asarray(weight, dtype=F32) / F32(scale), dtype)


def residual_add(a, b, dtype="f16"):
    """block_kernel.cu:7-17 with scale==1: c = T(a + b) (add performed in T)."""
    return _t(np.asarray(a, dtype=F32) + np.asarray(b, dtype=F32), dtype)


def add_then_rmsnorm(a, b, weight, eps, dtype="f16"):
    """Single-stream decode order (block.cpp:124-131): h = T(a+b); y = rmsnorm(h)."""
    h = residual_add(a, b, dtype)
    return h, rmsnorm(h, weight, eps, 1.0, dtype)


# ----------------------------------------------------------------------------
# RoPE
# ----------------------------------------------------------------------------
def rope_inv_freq(dim_head, theta, llama3=None):
    """rope_preparer.cu:49-69 and :124-161.  llama3 = dict(factor, low, high, orig) or None.
    Returns inv_freq for i in [0, dim_head/2) in fp32 (powf semantics)."""
    i = np.arange(dim_head // 2, dtype=F32)
    inv = np.power(F32(theta), -(i * F32(2)) / F32(dim_head)).astype(F32)
    if llama3:
        factor, low, high, orig = (F32(llama3[k]) for k in ("factor", "low", "high", "orig"))
        low_wl = orig / low
        high_wl = orig / high
        wl = F32(2.0) * F32(3.141592653589793) / inv
        smooth = (orig / wl - low) / (high - low)
        mid = (F32(1.0) - smooth) * inv / factor + smooth * inv
        inv = np.where(wl < high_wl, inv, np.where(wl > low_wl, inv / factor, mid)).astype(F32)
    return inv


def rope_cos_sin(pos, dim_head, theta, llama3=None, neox=True):
    """cos/sin tables fp32 (T, dim_head); column c uses i = c mod d/2 (neox) or c//2."""
    inv = rope_inv_freq(dim_head, theta, llama3)
    cols = np.arange(dim_head)
    idx = np.where(cols < dim_head // 2, cols, cols - dim_head // 2) if neox else cols // 2
    freq = np.asarray(pos, dtype=F32)[:, None] * inv[idx][None, :]
    # the reference calls double-precision cos()/sin() on a float argument, stores float
    return np.cos(freq.astype(np.float64)).astype(F32), np.sin(freq.astype(np.float64)).astype(F32)


def rope_apply(x, cos, sin, neox=True, dtype="f16"):
    """rope_common.cuh:13-34.  x (T, H, d) values in T; returns T-rounded result."""
    x = np.asarray(x, dtype=F32)
    d = x.shape[-1]
    h = d // 2
    c = cos[:, None, :]
    s = sin[:, None, :]
    if neox:
        rot = np.concatenate([-x[..., h:], x[..., :h]], axis=-1)
    else:
        rot = np.empty_like(x)
        rot[..., 0::2] = -x[..., 1::2]
        rot[..., 1::2] = x[..., 0::2]
    return _t(x * c + rot * s, dtype)


def split_qkv_rope(qkv, cos, sin, num_heads, num_kv_heads, dim_head, neox=True, dtype="f16"):
    """rotary_embedding_fuse_cache.cu:23-63: (T, (Hq+2Hkv)*d) -> q (T,Hq*d), k, v; RoPE on q,k."""
    t = qkv.shape[0]
    x = np.asarray(qkv, dtype=F32).reshape(t, num_heads + 2 * num_kv_heads, dim_head)
    q = rope_apply(x[:, :num_heads], cos, sin, neox, dtype)
    k = rope_apply(x[:, num_heads:num_heads + num_kv_heads], cos, sin, neox, dtype)
    v = x[:, num_heads + num_kv_heads:]
    return (q.reshape(t, -1), k.reshape(t, -1), np.ascontiguousarray(v).reshape(t, -1))


# ----------------------------------------------------------------------------
# activations
# ----------------------------------------------------------------------------
def silu(x):
    x = np.asarray(x, dtype=F32)
    return x / (F32(1.0) + np.exp(-x))


def gelu(x):
    x = np.asarray(x, dtype=F32)
    return F32(0.5) * x * (F32(1.0) + np.tanh(F32(0.7978845608028654) * x * (F32(1.0) + F32(0.044715) * x * x)))


def silu_mul(gate, up, dtype="f16"):
    """activation_kernel.cu:71-80: inp = T(silu(float(inp)) * float(in2)) on T-rounded inputs."""
    return _t(silu(_t(gate, dtype)) * _t(up, dtype), dtype)


# ----------------------------------------------------------------------------
# decode attention over per-task ragged KV buffers
# ----------------------------------------------------------------------------
def decode_attention(q, k_bufs, v_bufs, buf_lens, masks, scale, m_query, dtype="f16"):
    """attention_kernel.cu:674-725 + 434-489.

    q       (B, len_q, H_q, d)        values in T
    k_bufs  list of B arrays (len_buf_b, H_kv, d)   (BSHD layout)
    masks   list of B arrays (len_q, len_buf_b) int8
    returns (B, len_q, H_q, d) in T.
    logit = mask ? scale*(q.k) : -inf ; m = max ; e = exp(logit-m) ; sum = 1e-20 + sum(e) ;
    p = e/sum ; o = sum p*v in fp32.
    """
    q = np.asarray(q, dtype=F32)
    b, len_q, hq, d = q.shape
    out = np.zeros_like(q)
    for bi in range(b):
        lb = int(buf_lens[bi])
        k = np.asarray(k_bufs[bi], dtype=F32)[:lb]
        v = np.asarray(v_bufs[bi], dtype=F32)[:lb]
        msk = np.asarray(masks[bi]).reshape(len_q, lb) != 0
        for qi in range(len_q):
            for h in range(hq):
                hk = h // m_query
                logit = (k[:, hk, :] @ q[bi, qi, h]) * F32(scale)
                logit = np.where(msk[qi], logit, -np.inf).astype(F32)
                m = max(F32(-1e20), logit.max()) if lb else F32(-1e20)
                e = np.exp(logit - m).astype(F32)
                ssum = F32(1e-20) + e.sum(dtype=F32)
                p = e / ssum
                out[bi, qi, h] = p @ v[:, hk, :]
    return _t(out, dtype)


def split_kv_combine(partial_o, local_max, local_sum):
    """attention_kernel.cu:881-923: partial_o (S, d) each normalized by its local sum;
    w_i = sum_i*exp(m_i-M) / sum_j sum_j*exp(m_j-M)."""
    m = np.max(local_max)
    s1 = np.exp(local_max - m)
    g = (local_sum * s1).sum()
    w = local_sum / g * s1
    return (partial_o * w[:, None]).sum(0)


def kv_append(k_buf, v_buf, k_new, v_new, placement):
    """ragged_buffer_kernel.cu:194-222 (BSHD): buf[placement[i]] = new[i]; placement<0 skipped."""
    for i, p in enumerate(placement):
        if p >= 0:
            k_buf[p] = k_new[i]
            v_buf[p] = v_new[i]


# ----------------------------------------------------------------------------
# INT8 / FP8 activation quantization
# ----------------------------------------------------------------------------
def int8_quant_per_token(x):
    """quant_kernel.cu:15-47: scale = absmax/127 ; q = int8(nearbyint(x * (127/absmax))).
    An all-zero row gives 0*inf = NaN, which the device float->int8 conversion turns into 0 (scale 0)."""
    x = np.asarray(x, dtype=F32)
    amax = np.abs(x).max(-1, keepdims=True).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        bs = F32(127.0) / amax
        r = np.rint(x * bs)
    q = np.where(np.isnan(r), 0, r).astype(np.int8)
    return q, (amax / F32(127.0)).reshape(-1).astype(F32)


def rmsnorm_quant(x, weight, eps, scale=1.0, dtype="f16"):
    """layernorm_quant / fuse_layernorm_rms_quant (quant_kernel.cu:106-151): returns (y in T as f32, q int8, qscale).
    absmax of x*w is rounded through T (blockReduceMax<T>), 127.0/absmax is a double division rounded to float,
    the int8 twin quantises x*w/scale WITHOUT rsqrt and the scale carries rsqrt."""
    x = np.asarray(x, dtype=F32)
    w = np.asarray(weight, dtype=F32)
    d = x.shape[-1]
    vw = (x * w).astype(F32)
    amax = _t(np.abs(vw).max(-1, keepdims=True), dtype)
    rs = (F32(1.0) / np.sqrt((x.astype(np.float64) ** 2).sum(-1, keepdims=True) / d + eps)).astype(F32)
    with np.errstate(divide="ignore"):
        bs = (127.0 / amax.astype(np.float64)).astype(F32)
    v = (vw / F32(scale)).astype(F32)
    y = _t(v * rs, dtype)
    with np.errstate(invalid="ignore"):
        r = np.rint((v * bs).astype(F32))
    q = np.where(np.isnan(r), 0, r).astype(np.int8)
    qscale = ((amax * rs).astype(F32).astype(np.float64) / 127.0).astype(F32).reshape(-1)
    return y, q, qscale


def int8_weight_quant_per_row(w):
    """linear.cpp:521-550 (AutoInt8): per output-row absmax int8 at load."""
    return int8_quant_per_token(w)


def int8_scale_back(acc_i32, scale_x, scale_y, dtype="f16"):
    """quant_kernel.cu:231-246: y = T(float(acc) * s_x[m] * s_w[n])."""
    acc = np.asarray(acc_i32).astype(F32)
    return _t(acc * np.asarray(scale_x, F32)[:, None] * np.asarray(scale_y, F32)[None, :], dtype)


def int8_linear(x, w_q, w_scale, dtype="f16", bias=None):
    """Int8Linear::forward (linear.cpp:560-636): quant -> s32 gemm -> scale back (-> add_bias in T, :631-633)."""
    xq, xs = int8_quant_per_token(x)
    acc = xq.astype(np.int32) @ np.asarray(w_q).astype(np.int32).T
    y = int8_scale_back(acc, xs, w_scale, dtype)
    if bias is not None:
        y = _t(y + np.asarray(bias, F32), dtype)
    return y


E4M3_MAX = 448.0


def e4m3_round(x):
    """Round fp32 values to the nearest OCP e4m3fn value (saturating, RNE), returned as fp32."""
    x = np.asarray(x, dtype=np.float64)
    s = np.sign(x)
    a = np.minimum(np.abs(x), E4M3_MAX)
    out = np.zeros_like(a)
    nz = a > 0
    e = np.floor(np.log2(np.where(nz, a, 1.0)))
    e = np.maximum(e, -6.0)                       # subnormal exponent floor (2^-6, 3 mantissa bits)
    q = np.power(2.0, e - 3)                      # spacing
    out = np.rint(a / q) * q                      # np.rint = RNE
    out = np.minimum(out, E4M3_MAX)
    return (s * np.where(nz, out, 0.0)).astype(F32)


def e4m3_decode(b):
    """OCP e4m3fn byte -> fp32 value (0x7f/0xff = NaN)."""
    b = np.asarray(b, dtype=np.uint8).astype(np.int32)
    sign = np.where(b & 0x80, -1.0, 1.0)
    e = (b >> 3) & 0xF
    m = b & 7
    val = np.where(e == 0, m * 2.0 ** -9, (1.0 + m / 8.0) * np.exp2(e.astype(np.float64) - 7))
    val = np.where((e == 15) & (m == 7), np.nan, val)
    return (sign * val).astype(F32)


def fp8_quant_per_tensor(x, max_e4m3=E4M3_MAX, dtype="f16"):
    """fp8_util.cu:110-147,176-228: scale = max|x| / 448 over the whole tensor; q = e4m3_rn_satfinite(h) where
    h = x_f16 * half(1/scale) rounded in fp16 for fp16 inputs (:77-80) and h = half(float(x) * (1/scale)) for bf16
    inputs (:74-76).  Returns (values of q as fp32, scale)."""
    x = np.asarray(x, dtype=F32)
    scale = F32(np.abs(x).max()) / F32(max_e4m3)
    inv = F32(1.0) / scale
    if dtype == "f16":
        h = (x.astype(np.float16).astype(F32) * np.float16(inv).astype(F32)).astype(np.float16)
    else:
        h = (x * inv).astype(F32).astype(np.float16)
    return e4m3_round(h.astype(F32)), scale


def fp8_linear(x, w_fp8_vals, w_scale, dtype="f16", bias=None):
    """Fp8Linear::forward (linear.cpp:1660-1695): y = T((xq @ wq^T) * s_x * s_w), fp32 accumulate."""
    xq, xs = fp8_quant_per_tensor(x, dtype=dtype)
    acc = xq.astype(np.float64) @ np.asarray(w_fp8_vals, dtype=np.float64).T
    y = acc * np.float64(xs * F32(w_scale))
    if bias is not None:
        y = y + np.asarray(bias, dtype=np.float64)
    return _t(y.astype(F32), dtype)


# ----------------------------------------------------------------------------
# int8 TP all-reduce (group 32)
# ----------------------------------------------------------------------------
def quant_group_32(x, dtype="f16"):
    """quant_reduce_kernel.cu:14-38: x (..., 32) in T.  absmax reduced IN T; q = int8(nearbyint(v*127/absmax));
    scale = T(absmax/127)."""
    x = np.asarray(x, dtype=F32)
    amax = _t(np.abs(x).max(-1, keepdims=True), dtype)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.rint(x * F32(127.0) / amax)
    q = np.nan_to_num(q, nan=0.0).astype(np.int8)          # reference is NaN here (0/0) -- UB cast
    return q, _t(amax / F32(127.0), dtype).reshape(x.shape[:-1])


def dequant_sum_quant_g32(my, q_others, scale_others, dtype="f16"):
    """quant_reduce_kernel.cu:243-274: sum = my + sum_r q_r*s_r (fp32, r ascending); requant g32."""
    s = np.asarray(my, dtype=F32).copy()
    for r in range(len(q_others)):
        s = s + q_others[r].astype(F32) * np.asarray(scale_others[r], dtype=F32)[..., None]
    return quant_group_32(s, dtype)


def allreduce_int8_reference(partials, dtype="f16"):
    """model_context.cpp:244-326 simulated for WS ranks.  partials: list of WS arrays (T, D) in T.
    Returns the dequantized (T, D) result every rank ends with (step 4, dequant_group_32)."""
    ws = len(partials)
    shape = partials[0].shape
    numel = partials[0].size
    m = numel // ws // 32
    g = [np.asarray(p, dtype=F32).reshape(ws, m, 32) for p in partials]
    sent = [quant_group_32(g[r], dtype) for r in range(ws)]          # every rank quantizes all chunks
    q_sum = np.zeros((ws, m, 32), dtype=np.int8)
    s_sum = np.zeros((ws, m), dtype=F32)
    for r in range(ws):
        qo, so = [], []
        for i in range(ws - 1):
            src = (r + i + 1) % ws                                    # model_context.cpp:279
            qo.append(sent[src][0][r])
            so.append(sent[src][1][r])
        q_sum[r], s_sum[r] = dequant_sum_quant_g32(g[r][r], qo, so, dtype)
    out = q_sum.astype(F32) * s_sum[..., None]                        # dequant_group_32
    return _t(out, dtype).reshape(shape)


def allreduce_exact(partials, dtype="f16"):
    """fp32 sum of the partials rounded to T (what ncclAllReduce(sum) approximates)."""
    s = np.zeros(partials[0].shape, dtype=F32)
    for p in partials:
        s = s + np.asarray(p, dtype=F32)
    return _t(s, dtype)


def allreduce_int8_one_shot(partials, dtype="f16"):
    """The one-shot variant our NVLink kernel implements (zhilight_b200/csrc/comm.cu): every rank's contribution is
    quantised ONCE with quant_group_32 and all ranks add the same ws dequantised vectors in rank order in fp32."""
    acc = np.zeros(partials[0].size, dtype=F32).reshape(-1, 32)
    for p in partials:
        q, s = quant_group_32(np.asarray(p, dtype=F32).reshape(-1, 32), dtype)
        acc = acc + q.astype(F32) * np.asarray(s, dtype=F32)[:, None]
    return _t(acc, dtype).reshape(partials[0].shape)
