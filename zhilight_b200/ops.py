"""Torch-tensor front end of the C-ABI (plumbing only: torch supplies device memory and streams).

Every function takes CUDA tensors, passes raw pointers to libzhilight_b200.so on the current stream and
returns torch tensors.  Names / argument meaning mirror the reference operator each one replaces.
"""
import ctypes

import torch

from . import _lib

F16, BF16, F32 = 0, 1, 2
EPI_NONE, EPI_SWIGLU, EPI_RESIDUAL, EPI_QKV_ROPE = 0, 1, 2, 3


def _dt(t):
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.bfloat16:
        return BF16
    if t.dtype == torch.float32:
        return F32
    raise _lib.ZLError(-2, "unsupported dtype %s" % t.dtype)


def _p(t):
    if t is None:
        return None
    if not t.is_cuda:
        raise _lib.ZLError(-1, "zhilight_b200 ops need CUDA tensors (no CPU fallback)")
    if not t.is_contiguous():
        raise _lib.ZLError(-1, "tensor must be contiguous")
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------ load-time transforms
def gptq_shuffle(qweight, q_perm=None):
    """nn::gptq::gptq_shuffle -- in place on (K/8, N) int32."""
    k8, n = qweight.shape
    scratch = torch.empty_like(qweight) if q_perm is not None else None
    _lib.call("zl_gptq_shuffle", _p(qweight), _p(q_perm), _p(scratch), k8 * 8, n, _stream())
    return qweight


def gptq_increase_zero(qzeros):
    _lib.call("zl_gptq_increase_zero", _p(qzeros), qzeros.numel(), _stream())
    return qzeros


def gptq_subtract8(words):
    _lib.call("zl_gptq_subtract8", _p(words), words.numel(), _stream())
    return words


def q4_to_q8(qzeros):
    r, c8 = qzeros.shape
    out = torch.empty((r, c8 * 8), dtype=torch.uint8, device=qzeros.device)
    _lib.call("zl_q4_to_q8", _p(qzeros), _p(out), qzeros.numel(), _stream())
    return out


def awq_un_shuffle(qzeros):
    _lib.call("zl_awq_un_shuffle", _p(qzeros), qzeros.shape[0], qzeros.shape[1], _stream())
    return qzeros


def awq_shuffle(qweight, use_exllama=True):
    k, n8 = qweight.shape
    out = torch.empty((k // 8, n8 * 8), dtype=qweight.dtype, device=qweight.device)
    _lib.call("zl_awq_shuffle", _p(qweight), _p(out), k, n8 * 8, int(use_exllama), _stream())
    return out


def transpose_2d(x):
    r, c = x.shape
    out = torch.empty((c, r), dtype=x.dtype, device=x.device)
    _lib.call("zl_transpose_2d", _p(x), _p(out), r, c, x.element_size(), _stream())
    return out


def gptq_to_k_major(qweight, qzeros, scales, is_awq=False):
    """Int4GPTQ::preprocess_weight + transpose_weight (linear.cpp:1139-1160, 1085-1099) on device.
    Consumes copies of the HF tensors; returns (qweight_km (N,K/8) i32, qzeros_km (N,G) u8, scales_km (N,G) f16)."""
    if is_awq:
        qw = awq_shuffle(qweight.contiguous(), True)
        qz = awq_un_shuffle(qzeros.clone())
    else:
        qw = gptq_shuffle(qweight.clone())
        qz = gptq_increase_zero(qzeros.clone())
    z8 = q4_to_q8(qz)
    return transpose_2d(qw), transpose_2d(z8), transpose_2d(scales.contiguous())


def act_order_perm(g_idx, group_size=128):
    """The act-order permutation of a desc_act checkpoint's g_idx (host int32 tensor, K), or None when g_idx is
    sequential.  Same order as the reference's argsort_cpu (linear.cpp:1010-1028): a stable bucket sort of k by group."""
    gi = torch.as_tensor(g_idx).cpu().to(torch.int64).reshape(-1)
    k = gi.numel()
    if torch.equal(gi, torch.arange(k) // group_size):
        return None
    if k % group_size or gi.min() < 0 or gi.max() >= k // group_size or \
            not bool((torch.bincount(gi, minlength=k // group_size) == group_size).all()):
        raise _lib.ZLError(-1, "malformed g_idx: every group of %d columns must appear exactly %d times"
                           % (group_size, group_size))
    return torch.sort(gi, stable=True).indices.to(torch.int32)


def gptq_to_k_major_act_order(qweight, qzeros, scales, g_idx, group_size=128):
    """gptq_to_k_major for a GPTQ checkpoint that may be act-order: returns (qweight_km, qzeros_km, scales_km, k_perm),
    the k-major tensors sequentialised with k_perm (make_sequential, q_gemm.cu:794-829) and k_perm itself (K int32 on the
    weights' device), or k_perm = None for a sequential g_idx.  A GEMM on these weights takes x[:, k_perm]."""
    perm = act_order_perm(g_idx, group_size) if g_idx is not None else None
    if perm is None:
        return gptq_to_k_major(qweight, qzeros, scales) + (None,)
    perm = perm.to(qweight.device)
    qw = gptq_shuffle(qweight.clone(), perm)
    z8 = q4_to_q8(gptq_increase_zero(qzeros.clone()))
    return transpose_2d(qw), transpose_2d(z8), transpose_2d(scales.contiguous()), perm


def gather_cols(x, perm, pdl=False):
    """zl_gather_cols_16: y[m, i] = x[m, perm[i]] for a 16-bit x (M, K) with unit column stride; perm (K) int32."""
    if x.element_size() != 2 or not x.is_floating_point():
        raise _lib.ZLError(-2, "gather_cols needs a 16-bit float x, got %s" % x.dtype)
    if x.dim() != 2 or x.stride(1) != 1:
        raise _lib.ZLError(-1, "gather_cols needs a 2-D x with unit column stride")
    if perm.dtype != torch.int32 or perm.numel() != x.shape[1]:
        raise _lib.ZLError(-1, "gather_cols needs perm as K int32 entries")
    m, k = x.shape
    y = torch.empty((m, k), dtype=x.dtype, device=x.device)
    _lib.call("zl_gather_cols_16", ctypes.c_void_p(x.data_ptr()), x.stride(0), _p(perm), _p(y), m, k, int(pdl),
              _stream())
    return y


def gptq_dequant_k_major(qweight_km, qzeros_km, scales_km):
    n, k8 = qweight_km.shape
    g = scales_km.shape[1]
    out = torch.empty((n, k8 * 8), dtype=torch.float16, device=qweight_km.device)
    _lib.call("zl_gptq_dequant_k_major", _p(qweight_km), _p(qzeros_km), _p(scales_km), _p(out), n, k8 * 8,
              (k8 * 8) // g, _stream())
    return out


def w4_pack(qweight_km, qzeros_km, scales_km, group_size=128, sym=False, row_map=None, variant=0):
    n_src, k8 = qweight_km.shape
    n = n_src if row_map is None else row_map.numel()
    k = k8 * 8
    nbytes = _lib.load().zl_w4_packed_bytes(n, k, group_size)
    if nbytes == 0:
        raise _lib.ZLError(-2, "unsupported ZLW4 shape N=%d K=%d group=%d" % (n, k, group_size))
    packed = torch.empty(nbytes, dtype=torch.uint8, device=qweight_km.device)
    _lib.call("zl_w4_pack_v", _p(qweight_km), _p(qzeros_km), _p(scales_km), _p(row_map), _p(packed), n, k, group_size,
              int(sym), int(variant), _stream())
    return packed


def w4_unpack(packed, n, k, group_size=128, variant=0):
    dev = packed.device
    qw = torch.empty((n, k // 8), dtype=torch.int32, device=dev)
    qz = torch.empty((n, k // group_size), dtype=torch.uint8, device=dev)
    sc = torch.empty((n, k // group_size), dtype=torch.float16, device=dev)
    _lib.call("zl_w4_unpack_v", _p(packed), _p(qw), _p(qz), _p(sc), n, k, group_size, int(variant), _stream())
    return qw, qz, sc


def swiglu_row_map(f, device):
    p = torch.arange(2 * f, device=device, dtype=torch.int32)
    tile, r = p // 16, p % 16
    return torch.where(r < 8, tile * 8 + r, f + tile * 8 + (r - 8)).to(torch.int32).contiguous()


# ------------------------------------------------------------------ compute
def w4a16_gemm(x, packed, n, k, group_size=128, bias=None, residual=None, epilogue=EPI_NONE, pdl=False, out=None):
    """nn::gptq::gptq_gemm_k_major (GEMV path) on the ZLW4 layout."""
    if x.dtype != torch.float16:
        raise _lib.ZLError(-2, "A must be half")      # q_gemm_k_major.cu:989
    m = x.shape[0]
    n_out = n // 2 if epilogue == EPI_SWIGLU else n
    if out is None:
        out = torch.empty((m, n_out), dtype=torch.float16, device=x.device)
    _lib.call("zl_w4a16_gemm", _p(x), x.stride(0), _p(packed), _p(bias), _p(residual), _p(out), m, n, k, group_size,
              epilogue, int(pdl), _stream())
    return out


def _dp(t):
    return t.data_ptr() if t is not None else None


def qkv_rope_row_map(n_heads_total, dim_head, device):
    m = torch.empty(n_heads_total * dim_head, dtype=torch.int32, device=device)
    _lib.call("zl_qkv_rope_row_map", _p(m), n_heads_total, dim_head, _stream())
    return m


def gather_rows_16(src, row_map):
    dst = torch.empty(row_map.numel(), dtype=src.dtype, device=src.device)
    _lib.call("zl_gather_rows_16", _p(src), _p(row_map), _p(dst), row_map.numel(), _stream())
    return dst


def w4a16_gemm_fused(x, packed, n, k, group_size=128, bias=None, residual=None, epilogue=EPI_NONE, pdl=False, out=None,
                     ln_weight=None, eps=1e-5, rope=None, variant=0, k_perm=None, kv8=None):
    """zl_w4a16_gemm_fused.  rope = dict(cos, sin, token_batch, placement, k_bufs, v_bufs, num_heads, num_kv_heads,
    dim_head) for EPI_QKV_ROPE (returns q); bias must be in packed-row order.  k_perm (K int32, act-order): y = W . x[:, k_perm]
    with W packed from the sequentialised weights (exact-integer route only; elsewhere gather_cols first).
    kv8 = dict(sk_bufs, sv_bufs, stage, counters) with EPI_QKV_ROPE: k_bufs / v_bufs are uint8 code buffers and the epilogue
    quantises the K / V rows into them (int8 KV cache; exact-integer route only).  stage: fp16 (M, 2, H_kv, d) scratch,
    counters: int32 (M, 2, H_kv), zero before the first launch and left zero."""
    if x.dtype != torch.float16:
        raise _lib.ZLError(-2, "A must be half")
    m = x.shape[0]
    a = _lib.W4FusedArgs()
    a.x, a.ldx, a.packed, a.bias, a.residual = x.data_ptr(), x.stride(0), packed.data_ptr(), _dp(bias), _dp(residual)
    a.M, a.N, a.K, a.group_size, a.epilogue, a.pdl = m, n, k, group_size, epilogue, int(pdl)
    a.ln_weight, a.eps = _dp(ln_weight), eps
    a.variant = int(variant)
    a.k_perm = _dp(k_perm)
    keep = []
    if epilogue == EPI_QKV_ROPE:
        r = rope
        q = torch.empty((m, r["num_heads"] * r["dim_head"]), dtype=torch.float16, device=x.device)
        ka, va = _ptr_table(r["k_bufs"], x.device), _ptr_table(r["v_bufs"], x.device)
        keep += [ka, va]
        a.cos, a.sin, a.q_out = r["cos"].data_ptr(), r["sin"].data_ptr(), q.data_ptr()
        a.token_batch, a.placement = r["token_batch"].data_ptr(), r["placement"].data_ptr()
        a.k_addrs, a.v_addrs = ka.data_ptr(), va.data_ptr()
        a.num_heads, a.num_kv_heads, a.dim_head = r["num_heads"], r["num_kv_heads"], r["dim_head"]
        if kv8 is not None:
            ska, sva = _ptr_table(kv8["sk_bufs"], x.device), _ptr_table(kv8["sv_bufs"], x.device)
            keep += [ska, sva]
            a.kv_int8, a.scale_k_addrs, a.scale_v_addrs = 1, ska.data_ptr(), sva.data_ptr()
            a.kv8_stage, a.kv8_counters = kv8["stage"].data_ptr(), kv8["counters"].data_ptr()
        ret = q
    else:
        n_out = n // 2 if epilogue == EPI_SWIGLU else n
        if out is None:
            out = torch.empty((m, n_out), dtype=torch.float16, device=x.device)
        a.y = out.data_ptr()
        ret = out
    _lib.call("zl_w4a16_gemm_fused", ctypes.byref(a), _stream())
    if keep:
        torch.cuda.current_stream().synchronize()
    return ret


def dense_gemm_skinny(x, w, bias=None, out_dtype=None, pdl=False):
    m, k = x.shape
    n = w.shape[0]
    od = x.dtype if out_dtype is None else out_dtype
    out = torch.empty((m, n), dtype=od, device=x.device)
    _lib.call("zl_dense_gemm_skinny", _p(x), x.stride(0), _p(w), _p(bias), _p(out), m, n, k, _dt(x), _dt(out),
              int(pdl), _stream())
    return out


W8_INT8, W8_FP8 = 0, 1


def int8_quant_per_token(x, pdl=False):
    """int8_op::quant_calc_scale: returns (q int8 (M,K), scale f32 (M))."""
    m, k = x.shape
    q = torch.empty((m, k), dtype=torch.int8, device=x.device)
    scale = torch.empty((m,), dtype=torch.float32, device=x.device)
    _lib.call("zl_int8_quant_per_token", _p(x), x.stride(0), _p(q), _p(scale), m, k, _dt(x), int(pdl), _stream())
    return q, scale


def rmsnorm_quant(x, weight, eps, scale=1.0, pdl=False):
    """int8_op::layernorm_quant: returns (y, q int8, qscale f32 (T))."""
    t, d = x.shape
    y = torch.empty_like(x)
    q = torch.empty((t, d), dtype=torch.int8, device=x.device)
    qs = torch.empty((t,), dtype=torch.float32, device=x.device)
    _lib.call("zl_rmsnorm_quant", _p(x), _p(weight), _p(y), _p(q), _p(qs), t, d, eps, scale, _dt(x), int(pdl),
              _stream())
    return y, q, qs


def fp8_quant_per_tensor(x, pdl=False):
    """nn::fp8::dynamic_scaled_quant: returns (q uint8 holding e4m3 bits, scale f32 (1))."""
    q = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    scale = torch.empty((1,), dtype=torch.float32, device=x.device)
    _lib.call("zl_fp8_quant_per_tensor", _p(x), _p(q), _p(scale), x.numel(), _dt(x), int(pdl), _stream())
    return q, scale


def w8a8_gemm(xq, x_scale, w, w_scale, out_dtype, kind=W8_INT8, bias=None, pdl=False):
    m, k = xq.shape
    n = w.shape[0]
    y = torch.empty((m, n), dtype=out_dtype, device=xq.device)
    ws_dt = 2 if w_scale.dtype == torch.float32 else _dt(w_scale)
    _lib.call("zl_w8a8_gemm", _p(xq), _p(x_scale), _p(w), _p(w_scale), ws_dt, _p(bias), _p(y), m, n, k, kind,
              _dt(y), int(pdl), _stream())
    return y


def int8_linear(x, w_q, w_scale, bias=None, pdl=False):
    """Int8Linear::forward (linear.cpp:560-636) in two launches instead of three."""
    q, s = int8_quant_per_token(x, pdl)
    return w8a8_gemm(q, s, w_q, w_scale, x.dtype, W8_INT8, bias, pdl)


def fp8_linear(x, w_fp8, w_scale, bias=None, pdl=False):
    """Fp8Linear::forward (linear.cpp:1660-1695)."""
    q, s = fp8_quant_per_tensor(x, pdl)
    return w8a8_gemm(q, s, w_fp8, w_scale, x.dtype, W8_FP8, bias, pdl)


def fp8_quant_per_token_group(x, pdl=False):
    """nn::fp8::per_token_cast_to_fp8: returns (q uint8 (M,K) holding e4m3 bits, scale f32 (K/128, round_up(M, 4)))
    with one scale per (token, 128-column group), stored column-major like the reference."""
    m, k = x.shape
    ld = (m + 3) // 4 * 4
    q = torch.empty((m, k), dtype=torch.uint8, device=x.device)
    scale = torch.empty((k // 128 if k % 128 == 0 else 1, ld), dtype=torch.float32, device=x.device)
    _lib.call("zl_fp8_quant_per_token_group", _p(x), x.stride(0), _p(q), _p(scale), ld, m, k, _dt(x), int(pdl),
              _stream())
    return q, scale


def fp8_block_gemm(xq, x_scale, w, w_scale, out_dtype, pdl=False):
    """deep_gemm_fp8_block_h20_group: xq (M,K) e4m3 bytes, x_scale (K/128, ld) f32, w (N,K) e4m3,
    w_scale (ceil(N/128), K/128) f32 -> y (M,N) out_dtype."""
    m, k = xq.shape
    n = w.shape[0]
    y = torch.empty((m, n), dtype=out_dtype, device=xq.device)
    _lib.call("zl_fp8_block_gemm", _p(xq), _p(x_scale), x_scale.shape[-1], _p(w), _p(w_scale), _p(y), m, n, k, _dt(y),
              int(pdl), _stream())
    return y


def fp8_block_linear(x, w_fp8, w_scale_inv, pdl=False):
    """Fp8Block::forward (linear.cpp:1697-1960): per-token-group activation quant, then the block-scaled GEMM."""
    q, s = fp8_quant_per_token_group(x, pdl)
    return fp8_block_gemm(q, s, w_fp8, w_scale_inv, x.dtype, pdl)


def rmsnorm(x, weight, eps, scale=1.0, pdl=False):
    t, d = x.shape
    y = torch.empty_like(x)
    _lib.call("zl_rmsnorm", _p(x), _p(weight), _p(y), t, d, eps, scale, _dt(x), int(pdl), _stream())
    return y


def add_rmsnorm(a, b, weight, eps, scale=1.0, mode=0, pdl=False):
    t, d = a.shape
    out_sum = torch.empty_like(a)
    y = torch.empty_like(a)
    _lib.call("zl_add_rmsnorm", _p(a), _p(b), _p(weight), _p(out_sum), _p(y), t, d, eps, scale, mode, _dt(a),
              int(pdl), _stream())
    return out_sum, y


def element_add_scale(a, b, scale=1.0):
    c = torch.empty_like(a)
    _lib.call("zl_element_add_scale", _p(a), _p(b), _p(c), a.numel(), scale, _dt(a), _stream())
    return c


def gate_mul(gate, up, act="silu"):
    t, f = gate.shape
    out = torch.empty((t, f), dtype=gate.dtype, device=gate.device)
    # strided views are fine here: the C entry point takes row strides
    _lib.call("zl_gate_mul", ctypes.c_void_p(gate.data_ptr()), gate.stride(0),
              ctypes.c_void_p(up.data_ptr()) if up is not None else None, up.stride(0) if up is not None else 0, _p(out), f, t, f, 0 if act == "silu" else 1, _dt(gate), _stream())
    return out


def activation(x, act):
    """Linear::activate: silu / gelu in fp32, rounded to T."""
    return gate_mul(x, None, act)


def rope_cos_sin(pos, dim_head, theta, llama3=None, neox=True):
    t = pos.numel()
    cos = torch.empty((t, dim_head), dtype=torch.float32, device=pos.device)
    sin = torch.empty_like(cos)
    l3 = llama3 or {}
    _lib.call("zl_rope_cos_sin", _p(pos), _p(cos), _p(sin), t, dim_head, float(theta),
              float(l3.get("factor", 0.0)), float(l3.get("low", 1.0)), float(l3.get("high", 4.0)),
              float(l3.get("orig", 8192.0)), int(neox), _stream())
    return cos, sin


def rope_qk_cache(cos, sin, qkv, num_heads, num_kv_heads, dim_head, neox=True):
    t = qkv.shape[0]
    q = torch.empty((t, num_heads * dim_head), dtype=qkv.dtype, device=qkv.device)
    k = torch.empty((t, num_kv_heads * dim_head), dtype=qkv.dtype, device=qkv.device)
    v = torch.empty_like(k)
    _lib.call("zl_rope_qk_cache", _p(cos), _p(sin), _p(qkv), _p(q), _p(k), _p(v), t, num_heads, num_kv_heads,
              dim_head, int(neox), _dt(qkv), _stream())
    return q, k, v


def _ptr_table(tensors, device):
    return torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64, device=device)


def copy_to_rag_buffer2(placement, buf_lens, k_src, v_src, k_bufs, v_bufs, bshd=True):
    b, len_q, hkv, d = k_src.shape
    ka, va = _ptr_table(k_bufs, k_src.device), _ptr_table(v_bufs, k_src.device)
    _lib.call("zl_copy_to_rag_buffer2", _p(placement), _p(buf_lens), _p(k_src), _p(v_src), _p(ka), _p(va), b, len_q,
              hkv, d, int(bshd), _dt(k_src), _stream())
    torch.cuda.current_stream().synchronize()      # keep the pointer tables alive until the copy ran


def qkv_rope_append(cos, sin, qkv, token_batch, placement, k_bufs, v_bufs, num_heads, num_kv_heads, dim_head,
                    buf_lens=None, neox=True, bshd=True, pdl=False):
    t = qkv.shape[0]
    q = torch.empty((t, num_heads * dim_head), dtype=qkv.dtype, device=qkv.device)
    ka, va = _ptr_table(k_bufs, qkv.device), _ptr_table(v_bufs, qkv.device)
    _lib.call("zl_qkv_rope_append", _p(cos), _p(sin), _p(qkv), _p(q), _p(token_batch), _p(placement), _p(ka), _p(va),
              t, num_heads, num_kv_heads, dim_head, int(neox), int(bshd), _p(buf_lens), _dt(qkv), int(pdl), _stream())
    torch.cuda.current_stream().synchronize()
    return q


def decode_attention(q, buf_lens, k_bufs, v_bufs, mask, scale, max_len_buf, num_kv_heads, bshd=True, pdl=False):
    """nn::multi_query_attention_rag_buffer: q (B, len_q, H_q, d); k_bufs/v_bufs lists of per-task tensors."""
    b, len_q, hq, d = q.shape
    out = torch.empty_like(q)
    ws_bytes = _lib.load().zl_decode_attention_workspace_bytes(b, len_q, hq, d, max_len_buf)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=q.device)
    ka, va = _ptr_table(k_bufs, q.device), _ptr_table(v_bufs, q.device)
    _lib.call("zl_decode_attention", _p(q), _p(buf_lens), _p(ka), _p(va), _p(mask), float(scale), max_len_buf,
              _p(out), b, len_q, hq, num_kv_heads, d, int(bshd), _p(ws), ws_bytes, _dt(q), int(pdl), _stream())
    torch.cuda.current_stream().synchronize()
    return out


def mla_decode_attention(q, buf_lens, kv_bufs, mask, scale, max_len_buf, pdl=False):
    """MLA decode attention (nn::multi_query_attention_rag_buffer with dim_head 576): q (B, len_q, H, 576); kv_bufs a list
    of B per-task latent caches (len, 576) or (len, 1, 576), each row the key of every head and its first 512 elements
    the value; mask None or the int8 ragged concat of (len_q, len_buf_b).  Returns (B, len_q, H, 512)."""
    if q.dim() != 4 or q.shape[-1] != 576:
        raise _lib.ZLError(-1, "q must be (B, len_q, H, 576)")
    b, len_q, hq, _ = q.shape
    if len(kv_bufs) != b:
        raise _lib.ZLError(-1, "one latent cache per task expected")
    for t in kv_bufs:
        if not (t.dim() == 2 and t.shape[1] == 576) and not (t.dim() == 3 and t.shape[1:] == (1, 576)):
            raise _lib.ZLError(-1, "latent cache must be (len, 576) or (len, 1, 576)")
        if t.dtype != q.dtype:
            raise _lib.ZLError(-1, "latent cache dtype differs from q")
    out = torch.empty((b, len_q, hq, 512), dtype=q.dtype, device=q.device)
    ws_bytes = _lib.load().zl_mla_decode_attention_workspace_bytes(b, len_q, hq, max_len_buf)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=q.device)
    ka = _ptr_table(kv_bufs, q.device)
    _lib.call("zl_mla_decode_attention", _p(q), _p(buf_lens), _p(ka), _p(mask), float(scale), int(max_len_buf), _p(out), b,
              len_q, hq, _p(ws), ws_bytes, _dt(q), int(pdl), _stream())
    torch.cuda.current_stream().synchronize()
    return out


def varlen_attention(q, segments, k_bufs, v_bufs, scale, num_kv_heads, max_keys=None, pdl=False):
    """Causal variable-length attention: q (rows, H_q, d); segments (nseg, 4) int32 {task, row0, pos0, n} (host or device;
    rows row0 .. row0 + n - 1 are positions pos0 .. pos0 + n - 1 of task `task`, each attending keys 0 ..= its position);
    k_bufs / v_bufs lists of per-task (len, H_kv, d) tensors.  max_keys defaults to max(pos0 + n)."""
    if q.dim() != 3:
        raise _lib.ZLError(-1, "q must be (rows, H_q, d)")
    rows, hq, d = q.shape
    seg = torch.as_tensor(segments, dtype=torch.int32)
    if seg.dim() != 2 or seg.shape[1] != 4:
        raise _lib.ZLError(-1, "segments must be (nseg, 4) {task, row0, pos0, n}")
    if max_keys is None:
        max_keys = int((seg[:, 2] + seg[:, 3]).max().item())
    seg = seg.to(q.device).contiguous()
    nseg = seg.shape[0]
    out = torch.empty_like(q)
    ws_bytes = _lib.load().zl_varlen_attention_workspace_bytes(rows, nseg, hq, d, max_keys)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=q.device)
    ka, va = _ptr_table(k_bufs, q.device), _ptr_table(v_bufs, q.device)
    _lib.call("zl_varlen_attention", _p(q), _p(seg), nseg, rows, _p(ka), _p(va), float(scale), int(max_keys), _p(out), hq,
              num_kv_heads, d, _p(ws), ws_bytes, _dt(q), int(pdl), _stream())
    torch.cuda.current_stream().synchronize()
    return out


def decode_attention_kv8(q, buf_lens, k_bufs, v_bufs, sk_bufs, sv_bufs, mask, scale, max_len_buf, num_kv_heads, out_dtype=None,
                         pdl=False):
    """int8 KV cache attention: q (B, len_q, H_q, d) f16; k/v lists of (len_buf, H_kv, d) uint8; sk/sv lists of
    (len_buf, H_kv) fp32 scales."""
    b, len_q, hq, d = q.shape
    out = torch.empty(q.shape, dtype=out_dtype or q.dtype, device=q.device)
    ws_bytes = _lib.load().zl_decode_attention_workspace_bytes(b, len_q, hq, d, max_len_buf)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=q.device)
    tabs = [_ptr_table(x, q.device) for x in (k_bufs, v_bufs, sk_bufs, sv_bufs)]
    _lib.call("zl_decode_attention_kv8", _p(q), _p(buf_lens), _p(tabs[0]), _p(tabs[1]), _p(tabs[2]), _p(tabs[3]), _p(mask),
              float(scale), max_len_buf, _p(out), b, len_q, hq, num_kv_heads, d, _p(ws), ws_bytes, _dt(out), int(pdl),
              _stream())
    torch.cuda.current_stream().synchronize()
    return out


def kv_int8_quant_append(k_src, v_src, token_batch, placement, k_bufs, v_bufs, sk_bufs, sv_bufs):
    """k_src / v_src (T, H_kv, d) -> uint8 codes + fp32 scales scattered into the per-task caches."""
    t, hkv, d = k_src.shape
    tabs = [_ptr_table(x, k_src.device) for x in (k_bufs, v_bufs, sk_bufs, sv_bufs)]
    _lib.call("zl_kv_int8_quant_append", _p(k_src), _p(v_src), _p(token_batch), _p(placement), _p(tabs[0]), _p(tabs[1]),
              _p(tabs[2]), _p(tabs[3]), t, hkv, d, _dt(k_src), 0, _stream())
    torch.cuda.current_stream().synchronize()


def embedding(ids, table):
    t = ids.numel()
    out = torch.empty((t, table.shape[1]), dtype=table.dtype, device=table.device)
    _lib.call("zl_embedding", _p(ids), _p(table), _p(out), t, table.shape[1], table.shape[0], _dt(table), 0, _stream())
    return out


def argmax(logits):
    t, v = logits.shape
    out = torch.empty(t, dtype=torch.int32, device=logits.device)
    nb = _lib.load().zl_argmax_workspace_bytes(t)
    ws = torch.empty(nb, dtype=torch.uint8, device=logits.device)
    _lib.call("zl_argmax", _p(logits), _p(out), t, v, _p(ws), nb, 0, _stream())
    return out


def sample_params_array(params, n):
    """Host zl_sample_params_t[n] from one parameter dict (every task) or a list of n dicts / SampleParams;
    validated with zl_sample_check_params."""
    if isinstance(params, (dict, _lib.SampleParams)):
        params = [params] * n
    if len(params) != n:
        raise _lib.ZLError(-1, "need %d parameter sets, got %d" % (n, len(params)))
    arr = (_lib.SampleParams * n)(*[q if isinstance(q, _lib.SampleParams) else _lib.sample_params(**q) for q in params])
    _lib.call("zl_sample_check_params", ctypes.cast(arr, ctypes.c_void_p), n)
    return arr


def sample(logits, params, row_task=None, counter=None, history=None, pdl=False):
    """Sampled (or greedy) next token per row of fp32 logits (T, V), zl_sample's contract.  params: one dict of
    set_sampling's keywords for every row, or one per task (a list); row_task (T) int32 maps rows to tasks (default:
    row i -> task i); counter (T) int32 (default 0); history (tasks, ceil(V/32)) int32 bitmap, updated in place, or None."""
    t, v = logits.shape
    n_tasks = len(params) if isinstance(params, (list, tuple)) else (history.shape[0] if history is not None else t)
    arr = sample_params_array(params, n_tasks)
    dparams = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(logits.device)
    out = torch.empty(t, dtype=torch.int32, device=logits.device)
    hw = history.shape[1] if history is not None else 0
    _lib.call("zl_sample", _p(logits), t, v, _p(dparams), _p(row_task), _p(counter), _p(history), hw, _p(out), None, 0,
              int(pdl), _stream())
    return out
