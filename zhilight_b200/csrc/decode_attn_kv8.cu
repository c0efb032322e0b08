// Decode attention over an int8 KV cache (KV_CACHE_DTYPE=int8 of the reference) and the quantising KV append.
//
// Replaces KERNEL_mqa_rag_buffer_split_kv_quant + DEV_mul_qk_quant_h128 / DEV_mul_logit_scale / DEV_mul_score_v_v1
// (reference src/nn/attention/attention_kernel.cu:804-880, src/nn/attention/quant_attention.cuh:10-123) and the
// cache-side quantisation int8_op::quant_calc_scale(x, 127, 128) + copy_to_rag_buffer2 of Attention::attn_search_rag
// (src/nn/attention/attention.cpp:656-676, src/nn/quant/int8/quant_kernel.cu:15-47).
//
// Cache contract (BSHD): per task K / V buffers (len_buf, H_kv, d) uint8 = round(x * 127 / absmax) + 128 and
// scale buffers (len_buf, H_kv) fp32 = absmax / 127, one scale per (token, kv head).  q is fp16.
//   logit[key] = scale * scale_k[key] * sum_d q[d] * (k[key, d] - 128)         (mask ? ... : -inf)
//   out[d]     = sum_key softmax(logit)[key] * scale_v[key] * (v[key, d] - 128)
// Same CTA decomposition as k_decode_attn (decode_attn_prologue, attn_common.cuh): one CTA per (kv split, kv head
// group, task x query), the whole GQA group shares every cache byte; K bytes become exact fp16 integers (PRMT 0x64xx
// magic) and feed mma.sync with fp32 accumulation -- the reference multiplies and pair-adds in fp16
// (quant_attention.cuh:60-70), so ours is the closer one to the exact result.  Half the algorithmic bytes of the fp16 cache: 2 * H_kv * d * ctx + 8 * H_kv * ctx per task per layer.
#include "attn_common.cuh"
#include "kv8_quant.cuh"

namespace zl {

// 4 cache bytes -> 4 exact fp16 integers (u8 - 128): 0x64xx = 1024 + x, minus 1152
__device__ __forceinline__ void u8x4_to_h2x2(uint32_t b, uint32_t& h01, uint32_t& h23) {
    uint32_t a0 = __byte_perm(b, 0x64646464u, 0x4140), a1 = __byte_perm(b, 0x64646464u, 0x4342);
    const __half2 off = __float2half2_rn(1152.f);
    __half2 r0 = __hsub2(*reinterpret_cast<__half2*>(&a0), off), r1 = __hsub2(*reinterpret_cast<__half2*>(&a1), off);
    h01 = *reinterpret_cast<uint32_t*>(&r0);
    h23 = *reinterpret_cast<uint32_t*>(&r1);
}
// one cache byte -> float(u8) - 128 via the 2^23 magic
__device__ __forceinline__ float u8_to_f32(uint32_t word, int i) {
    const uint32_t sel = 0x7540u | (uint32_t)i;
    return __uint_as_float(__byte_perm(word, 0x4B000000u, sel)) - 8388736.f;
}

template <typename TO, int D>
__global__ void __launch_bounds__(kAttnThreads)
k_decode_attn_kv8(const __half* __restrict__ q, const int32_t* __restrict__ buf_lens, uint8_t* const* __restrict__ k_addrs,
                  uint8_t* const* __restrict__ v_addrs, float* const* __restrict__ sk_addrs,
                  float* const* __restrict__ sv_addrs, const int8_t* __restrict__ mask, float scale, TO* __restrict__ out,
                  float* __restrict__ part_o, float* __restrict__ part_m, float* __restrict__ part_l, int len_q,
                  int num_heads, int num_kv_heads, int m_query, int num_splits) {
    constexpr int NI = D / 32;                 // 8-byte chunks per lane per key row
    __shared__ __align__(16) float s_logit[8 * kAttnRowStride];
    __shared__ float s_sv[kAttnMaxRange];      // V scales of the split's keys
    __shared__ float s_m[8], s_l[8], s_w[8];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;

    const DecodeAttnItem cta = decode_attn_prologue(buf_lens, len_q, m_query, num_splits);
    const int hk = cta.hk, mq = cta.mq, k0 = cta.k0, k1 = cta.k1, n = max(0, k1 - k0);

    const size_t stride = (size_t)num_kv_heads * D;          // BSHD, bytes
    const uint8_t* kbase = k_addrs[cta.b] + (size_t)hk * D;
    const uint8_t* vbase = v_addrs[cta.b] + (size_t)hk * D;
    const float* skb = sk_addrs[cta.b] + hk;                  // (len_buf, H_kv)
    const float* svb = sv_addrs[cta.b] + hk;
    const int8_t* mrow = cta.mask_row(mask, buf_lens, len_q);

    // ---- phase 1: S = K.Q^T on tensor cores (K bytes -> exact fp16 integers) ----
    uint4 qf[NI];
    decode_attn_load_q<D>(qf, q, cta, num_heads, g, t);
    const int ntiles = (n + 15) >> 4;
    for (int tile = warp; tile < ntiles; tile += kAttnWarps) {
        const int ka_i = k0 + tile * 16 + g, kb_i = ka_i + 8;
        const int ra = min(ka_i, k1 - 1), rb = min(kb_i, k1 - 1);
        const uint8_t* pa = kbase + (size_t)ra * stride + t * 8;
        const uint8_t* pb = kbase + (size_t)rb * stride + t * 8;
        uint2 ka[NI], kb[NI];
#pragma unroll
        for (int i = 0; i < NI; ++i) {
            ka[i] = ld_cg_u2(pa + i * 32);
            kb[i] = ld_cg_u2(pb + i * 32);
        }
        const float sa = __ldcg(skb + (size_t)ra * num_kv_heads), sb = __ldcg(skb + (size_t)rb * num_kv_heads);
        if (t == 0) {   // the V scales ride along with the K loads, so that phase 2 reads them from shared memory
            s_sv[tile * 16 + g] = __ldcg(svb + (size_t)ra * num_kv_heads);
            s_sv[tile * 16 + g + 8] = __ldcg(svb + (size_t)rb * num_kv_heads);
        }
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < NI; ++i) {
            uint32_t a01, a23, a45, a67, b01, b23, b45, b67;
            u8x4_to_h2x2(ka[i].x, a01, a23);
            u8x4_to_h2x2(ka[i].y, a45, a67);
            u8x4_to_h2x2(kb[i].x, b01, b23);
            u8x4_to_h2x2(kb[i].y, b45, b67);
            const uint32_t f0[4] = {a01, b01, a23, b23};
            const uint32_t f1[4] = {a45, b45, a67, b67};
            mma_16816_f16(acc, f0, qf[i].x, qf[i].y, acc);
            mma_16816_f16(acc, f1, qf[i].z, qf[i].w, acc);
        }
        const bool va = ka_i < k1 && (!mrow || mrow[ka_i] != 0);
        const bool vb = kb_i < k1 && (!mrow || mrow[kb_i] != 0);
        const int la = tile * 16 + g;
        const float ninf = -INFINITY;
        if (2 * t < mq) {
            s_logit[(2 * t) * kAttnRowStride + la] = va ? acc[0] * sa * scale : ninf;
            s_logit[(2 * t) * kAttnRowStride + la + 8] = vb ? acc[2] * sb * scale : ninf;
        }
        if (2 * t + 1 < mq) {
            s_logit[(2 * t + 1) * kAttnRowStride + la] = va ? acc[1] * sa * scale : ninf;
            s_logit[(2 * t + 1) * kAttnRowStride + la + 8] = vb ? acc[3] * sb * scale : ninf;
        }
    }
    __syncthreads();

    // ---- phase 2: masked softmax statistics per head; the V scale is folded into the stored weights w = e * scale_v,
    // and s_w keeps the split's largest weight per head (floored at 1e-30 so that 1024 / s_w stays finite) ----
    for (int h = warp; h < mq; h += kAttnWarps) {
        float* row = s_logit + h * kAttnRowStride;
        float mx = -1e20f;
        for (int i = lane; i < n; i += 32) mx = fmaxf(mx, row[i]);
        mx = warp_max(mx);
        float sum = 0.f, wmax = 0.f;
        for (int i = lane; i < n; i += 32) {
            const float e = expf(row[i] - mx);
            const float w = e * s_sv[i];
            sum += e;
            row[i] = w;
            wmax = fmaxf(wmax, w);
        }
        sum = warp_sum(sum) + 1e-20f;
        wmax = warp_max(wmax);
        if (lane == 0) {
            s_m[h] = mx;
            s_l[h] = sum;
            s_w[h] = fmaxf(wmax, 1e-30f);
        }
    }
    __syncthreads();

    // ---- phase 3: O = (P * scale_v) . (V - 128) on the tensor cores (mma.sync m16n8k16, fp32 accumulate) ----
    // A = weights [head (8 of 16 rows) x 16 keys] as fp16 w * 2^10 / s_w: at most 1024, so a V row with a large absmax
    // cannot overflow fp16, and small weights stay normal numbers; s_w / 2^10 is multiplied back in when the accumulators
    // are written out.  B = V [16 keys x 8 columns] as exact fp16 integers.  A B fragment register holds TWO KEYS of one
    // column, V is stored key-major: lane (g, t) loads D/8 contiguous bytes (columns NJ g .. NJ g + NJ - 1) of its four keys 2t, 2t+1, 2t+8,
    // 2t+9 and byte-interleaves row pairs with PRMT; n-tile j column c then stands for column d = NJ c + j of V (any
    // permutation of the columns is as good as another -- it is undone when the accumulators are written out).
    constexpr int NJ = D / 8;                        // n-tiles = V columns per lane and key row
    constexpr int NW = NJ / 4;                       // 32-bit words of a lane's column chunk
    float o[NJ][4];
#pragma unroll
    for (int j = 0; j < NJ; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    const __half2 voff = __float2half2_rn(1152.f);   // 1024 (magic) + 128 (zero point of the cache)
    const float wenc = g < mq ? 1024.f / s_w[g] : 0.f;
    for (int tile = warp; tile < ntiles; tile += kAttnWarps) {
        const int kb = tile * 16;                    // first key of the tile, relative to k0
        uint32_t vw[4][NW];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int kk = kb + 2 * t + (r & 1) + (r >> 1) * 8;
#pragma unroll
            for (int w = 0; w < NW; ++w) vw[r][w] = 0x80808080u;          // out of range: v - 128 = 0
            if (kk < n) {
                const uint8_t* src = vbase + (size_t)(k0 + kk) * stride + g * NJ;
                if constexpr (NW == 4) {
                    const uint4 v = ld_cg_u4(src);
                    vw[r][0] = v.x, vw[r][1] = v.y, vw[r][2] = v.z, vw[r][3] = v.w;
                } else {
                    const uint2 v = ld_cg_u2(src);
                    vw[r][0] = v.x, vw[r][1] = v.y;
                }
            }
        }
        uint32_t af[4] = {0u, 0u, 0u, 0u};
        if (g < mq) {
            const float* pr = s_logit + g * kAttnRowStride + kb + 2 * t;
            const float2 p0 = *reinterpret_cast<const float2*>(pr), p1 = *reinterpret_cast<const float2*>(pr + 8);
            const bool in0 = kb + 2 * t < n, in1 = kb + 2 * t + 1 < n, in2 = kb + 2 * t + 8 < n, in3 = kb + 2 * t + 9 < n;
            const __half2 h0 = __floats2half2_rn(in0 ? p0.x * wenc : 0.f, in1 ? p0.y * wenc : 0.f);
            const __half2 h1 = __floats2half2_rn(in2 ? p1.x * wenc : 0.f, in3 ? p1.y * wenc : 0.f);
            af[0] = *reinterpret_cast<const uint32_t*>(&h0);   // (head g, keys 2t, 2t+1)
            af[2] = *reinterpret_cast<const uint32_t*>(&h1);   // (head g, keys 2t+8, 2t+9); rows g+8 (a1, a3) stay zero
        }
#pragma unroll
        for (int wq = 0; wq < NW; ++wq) {
            // bytes 4 wq .. 4 wq + 3 of the key pairs -> {k, k+1} interleaved
            const uint32_t lo01 = __byte_perm(vw[0][wq], vw[1][wq], 0x5140), hi01 = __byte_perm(vw[0][wq], vw[1][wq], 0x7362);
            const uint32_t lo23 = __byte_perm(vw[2][wq], vw[3][wq], 0x5140), hi23 = __byte_perm(vw[2][wq], vw[3][wq], 0x7362);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const uint32_t s01 = e < 2 ? lo01 : hi01, s23 = e < 2 ? lo23 : hi23;
                const uint32_t sel = (e & 1) ? 0x4342u : 0x4140u;
                uint32_t b0 = __byte_perm(s01, 0x64646464u, sel), b1 = __byte_perm(s23, 0x64646464u, sel);
                __half2 hb0 = __hsub2(*reinterpret_cast<__half2*>(&b0), voff), hb1 = __hsub2(*reinterpret_cast<__half2*>(&b1), voff);
                mma_16816_f16(o[wq * 4 + e], af, *reinterpret_cast<uint32_t*>(&hb0), *reinterpret_cast<uint32_t*>(&hb1), o[wq * 4 + e]);
            }
        }
    }
    __syncthreads();
    float* s_red = s_logit;   // [warp][h][D]
    if (g < mq) {
        // accumulator (n-tile j, column c = 2t + i) = head g, V column NJ c + j; rows g + 8 (o[j][2..3]) are padding
        const float wdec = s_w[g] * (1.f / 1024.f);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            s_red[(warp * 8 + g) * D + NJ * (2 * t) + j] = o[j][0] * wdec;
            s_red[(warp * 8 + g) * D + NJ * (2 * t + 1) + j] = o[j][1] * wdec;
        }
    }
    __syncthreads();
    decode_attn_reduce_store<TO, D>(cta, s_red, s_m, s_l, num_heads, num_splits, out, part_o, part_m, part_l);
}

// quant_calc_scale(x, 127, 128) of one (token, kv head) row + scatter into the task's cache at placement (BSHD):
// grid (B * len_q, H_kv, 2 [k, v]), block d
template <typename T>
__global__ void k_kv8_quant_append(const T* __restrict__ k_src, const T* __restrict__ v_src, const int32_t* __restrict__ token_batch,
                                   const int32_t* __restrict__ placement, uint8_t* const* __restrict__ k_addrs,
                                   uint8_t* const* __restrict__ v_addrs, float* const* __restrict__ sk_addrs,
                                   float* const* __restrict__ sv_addrs, int num_kv_heads) {
    __shared__ float s_max[32];
    const int tok = blockIdx.x, hk = blockIdx.y, is_v = blockIdx.z, d = blockDim.x, c = threadIdx.x;
    pdl_trigger();
    pdl_wait();
    const T* src = (is_v ? v_src : k_src) + ((size_t)tok * num_kv_heads + hk) * d;
    const float x = to_f32<T>(src[c]);
    float amax = warp_max(fabsf(x));
    if ((c & 31) == 0) s_max[c >> 5] = amax;
    __syncthreads();
    amax = 0.f;
    for (int w = 0; w < (d + 31) / 32; ++w) amax = fmaxf(amax, s_max[w]);
    const int pl = placement[tok];
    if (pl < 0) return;
    const int b = token_batch[tok];
    uint8_t* dst = (is_v ? v_addrs : k_addrs)[b] + ((size_t)pl * num_kv_heads + hk) * d;
    dst[c] = kv8_code(x, kv8_row_mul(amax));
    if (c == 0) (is_v ? sv_addrs : sk_addrs)[b][(size_t)pl * num_kv_heads + hk] = kv8_row_scale(amax);
}

// dense form of the same quantisation: int8_op::quant_calc_scale(x, 127, 128) on (M, K) rows -> uint8 codes + fp32 scales
template <typename T>
__global__ void k_int8_quant_rows_u8(const T* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ scale, int K) {
    __shared__ float s_max[32];
    const size_t off = (size_t)blockIdx.x * K;
    float amax = 0.f;
    for (int i = threadIdx.x; i < K; i += blockDim.x) amax = fmaxf(amax, fabsf(to_f32<T>(x[off + i])));
    amax = warp_max(amax);
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = amax;
    __syncthreads();
    amax = 0.f;
    for (int w = 0; w < (int)(blockDim.x + 31) / 32; ++w) amax = fmaxf(amax, s_max[w]);
    const float mul = kv8_row_mul(amax);
    for (int i = threadIdx.x; i < K; i += blockDim.x) q[off + i] = kv8_code(to_f32<T>(x[off + i]), mul);
    if (threadIdx.x == 0) scale[blockIdx.x] = kv8_row_scale(amax);
}

}  // namespace zl

using namespace zl;

extern "C" int zl_int8_quant_rows_u8(const void* x, void* q, float* scale, int M, int K, int dtype, zl_stream_t stream) {
    ZL_CHECK_ARG(x && q && scale && M > 0 && K > 0);
    ZL_CHECK_SUPPORTED(dtype == ZL_F16 || dtype == ZL_BF16);
    const int threads = K >= 1024 ? 1024 : ((K + 31) / 32) * 32;
    if (dtype == ZL_F16)
        k_int8_quant_rows_u8<__half><<<M, threads, 0, stream>>>((const __half*)x, (uint8_t*)q, scale, K);
    else
        k_int8_quant_rows_u8<__nv_bfloat16><<<M, threads, 0, stream>>>((const __nv_bfloat16*)x, (uint8_t*)q, scale, K);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_kv_int8_quant_append(const void* k_src, const void* v_src, const int32_t* token_batch,
                                       const int32_t* placement, void* const* k_addrs, void* const* v_addrs,
                                       void* const* scale_k_addrs, void* const* scale_v_addrs, int T, int num_kv_heads,
                                       int dim_head, int dtype, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(k_src && v_src && token_batch && placement && k_addrs && v_addrs && scale_k_addrs && scale_v_addrs);
    ZL_CHECK_ARG(T > 0 && num_kv_heads > 0 && dim_head > 0 && dim_head <= 1024 && dim_head % 32 == 0);
    ZL_CHECK_SUPPORTED(dtype == ZL_F16 || dtype == ZL_BF16);
    dim3 grid(T, num_kv_heads, 2), block(dim_head);
    if (dtype == ZL_F16)
        ZL_CHECK_CUDA(launch(k_kv8_quant_append<__half>, grid, block, 0, stream, pdl != 0, (const __half*)k_src,
                             (const __half*)v_src, token_batch, placement, (uint8_t* const*)k_addrs, (uint8_t* const*)v_addrs,
                             (float* const*)scale_k_addrs, (float* const*)scale_v_addrs, num_kv_heads));
    else
        ZL_CHECK_CUDA(launch(k_kv8_quant_append<__nv_bfloat16>, grid, block, 0, stream, pdl != 0, (const __nv_bfloat16*)k_src,
                             (const __nv_bfloat16*)v_src, token_batch, placement, (uint8_t* const*)k_addrs,
                             (uint8_t* const*)v_addrs, (float* const*)scale_k_addrs, (float* const*)scale_v_addrs,
                             num_kv_heads));
    return ZL_OK;
}

extern "C" int zl_decode_attention_kv8(const void* q, const int32_t* buf_lens, void* const* k_addrs, void* const* v_addrs,
                                       void* const* scale_k_addrs, void* const* scale_v_addrs, const int8_t* mask,
                                       float scale, int max_len_buf, void* out, int B, int len_q, int num_heads,
                                       int num_kv_heads, int dim_head, void* workspace, size_t workspace_bytes,
                                       int out_dtype, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(q && buf_lens && k_addrs && v_addrs && scale_k_addrs && scale_v_addrs && out);
    ZL_CHECK_ARG(B > 0 && len_q > 0 && max_len_buf > 0 && num_heads > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0);
    ZL_CHECK_SUPPORTED(dim_head == 128 || dim_head == 64);     // the reference: 128 only (attention_kernel.cu:1314)
    ZL_CHECK_SUPPORTED(out_dtype == ZL_F16 || out_dtype == ZL_BF16);
    const int m_query = num_heads / num_kv_heads;
    const int splits = attn_num_splits(B, len_q, num_kv_heads, m_query, max_len_buf);
    ZL_CHECK_SUPPORTED(splits <= kAttnMaxSplits);
    const size_t vheads = (size_t)B * len_q * num_heads;
    if (splits > 1) ZL_CHECK_ARG(workspace != nullptr && workspace_bytes >= attn_parts_bytes(vheads, splits, dim_head));
    const AttnParts part = attn_parts(workspace, vheads, splits, dim_head);
    dim3 grid(splits, num_kv_heads * ((m_query + 7) / 8), B * len_q), block(kAttnThreads);
#define ZL_A8_LAUNCH(TO, DD)                                                                                         \
    ZL_CHECK_CUDA(launch(k_decode_attn_kv8<TO, DD>, grid, block, 0, stream, pdl != 0, (const __half*)q, buf_lens,    \
                         (uint8_t* const*)k_addrs, (uint8_t* const*)v_addrs, (float* const*)scale_k_addrs,           \
                         (float* const*)scale_v_addrs, mask, scale, (TO*)out, part.o, part.m, part.l, len_q,         \
                         num_heads, num_kv_heads, m_query, splits));                                                 \
    ZL_CHECK_CUDA(launch_attn_combine(part, vheads, DD, (TO*)out, splits, stream, pdl != 0));
    if (out_dtype == ZL_F16) {
        if (dim_head == 128) { ZL_A8_LAUNCH(__half, 128) } else { ZL_A8_LAUNCH(__half, 64) }
    } else {
        if (dim_head == 128) { ZL_A8_LAUNCH(__nv_bfloat16, 128) } else { ZL_A8_LAUNCH(__nv_bfloat16, 64) }
    }
#undef ZL_A8_LAUNCH
    return ZL_OK;
}
