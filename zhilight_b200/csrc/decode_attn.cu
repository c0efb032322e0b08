// Batch decode attention over per-task ragged KV buffers (GQA/MQA), split-KV with LSE combine.
//
// Replaces nn::multi_query_attention_rag_buffer and its kernels KERNEL_mqa_rag_buffer1 /
// KERNEL_mqa_rag_buffer_split_kv / KERNEL_mqa_combine / the wmma KERNEL_mqa_rag_buffer
// (reference src/nn/attention/attention_kernel.cu:674-725, 730-923, 926-1017, 1252-1457).
//
// One CTA = (kv-split, kv-head, task x query).  The whole GQA group (<= 8 q-heads per pass) shares
// every K/V byte: K is read ONCE per kv-head straight into tensor-core A fragments (16 keys x 16 dims),
// Q is the B operand (16 dims x 8 heads), so S = K.Q^T needs no shuffles; softmax is the reference's
// exact two-pass fp32 form inside the split (mask ? scale*s : -inf, max seeded -1e20, sum seeded 1e-20);
// P.V runs on the tensor cores too, with fp32 accumulators.
// Splits are merged with the reference's LSE rule (attention_kernel.cu:881-923).
#include "attn_common.cuh"
#include "decode_attn_warp.cuh"

namespace zl {

template <typename T, int D>
__global__ void __launch_bounds__(kAttnThreads)
k_decode_attn(const T* __restrict__ q, const int32_t* __restrict__ buf_lens, T* const* __restrict__ k_addrs,
              T* const* __restrict__ v_addrs, const int8_t* __restrict__ mask, float scale,
              T* __restrict__ out, float* __restrict__ part_o, float* __restrict__ part_m,
              float* __restrict__ part_l, int len_q, int num_heads, int num_kv_heads, int m_query,
              int num_splits, int bshd) {
    constexpr int NI = D / 32;                 // 16-byte chunks per lane per key row
    __shared__ __align__(16) float s_logit[8 * kAttnRowStride];
    __shared__ float s_m[8], s_l[8];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;

    const DecodeAttnItem cta = decode_attn_prologue(buf_lens, len_q, m_query, num_splits);
    const int mq = cta.mq, k0 = cta.k0, k1 = cta.k1, n = max(0, k1 - k0);

    const size_t stride = bshd ? (size_t)num_kv_heads * D : (size_t)D;
    const size_t base = bshd ? (size_t)cta.hk * D : (size_t)cta.hk * cta.len_buf * D;
    const T* kbase = k_addrs[cta.b] + base;
    const T* vbase = v_addrs[cta.b] + base;
    const int8_t* mrow = cta.mask_row(mask, buf_lens, len_q);

    // ---- phase 1: S = K.Q^T on tensor cores ----
    uint4 qf[NI];
    decode_attn_load_q<D>(qf, q, cta, num_heads, g, t);
    const int ntiles = (n + 15) >> 4;
    for (int tile = warp; tile < ntiles; tile += kAttnWarps) {
        const int ka_i = k0 + tile * 16 + g, kb_i = ka_i + 8;
        const T* pa = kbase + (size_t)min(ka_i, k1 - 1) * stride + t * 8;
        const T* pb = kbase + (size_t)min(kb_i, k1 - 1) * stride + t * 8;
        uint4 ka[NI], kb[NI];
#pragma unroll
        for (int i = 0; i < NI; ++i) {
            ka[i] = ld_cg_u4(pa + i * 32);
            kb[i] = ld_cg_u4(pb + i * 32);
        }
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < NI; ++i) {
            const uint32_t a0[4] = {ka[i].x, kb[i].x, ka[i].y, kb[i].y};
            const uint32_t a1[4] = {ka[i].z, kb[i].z, ka[i].w, kb[i].w};
            mma_attn<T>(acc, a0, qf[i].x, qf[i].y);
            mma_attn<T>(acc, a1, qf[i].z, qf[i].w);
        }
        const bool va = ka_i < k1 && (!mrow || mrow[ka_i] != 0);
        const bool vb = kb_i < k1 && (!mrow || mrow[kb_i] != 0);
        const int la = tile * 16 + g;
        const float ninf = -INFINITY;
        if (2 * t < mq) {
            s_logit[(2 * t) * kAttnRowStride + la] = va ? acc[0] * scale : ninf;
            s_logit[(2 * t) * kAttnRowStride + la + 8] = vb ? acc[2] * scale : ninf;
        }
        if (2 * t + 1 < mq) {
            s_logit[(2 * t + 1) * kAttnRowStride + la] = va ? acc[1] * scale : ninf;
            s_logit[(2 * t + 1) * kAttnRowStride + la + 8] = vb ? acc[3] * scale : ninf;
        }
    }
    __syncthreads();

    // ---- phase 2: masked softmax statistics per head (attention_kernel.cu:434-489) ----
    for (int h = warp; h < mq; h += kAttnWarps) {
        float* row = s_logit + h * kAttnRowStride;
        float mx = -1e20f;
        for (int i = lane; i < n; i += 32) mx = fmaxf(mx, row[i]);
        mx = warp_max(mx);
        float sum = 0.f;
        for (int i = lane; i < n; i += 32) {
            const float e = expf(row[i] - mx);
            row[i] = e;
            sum += e;
        }
        sum = warp_sum(sum) + 1e-20f;
        if (lane == 0) {
            s_m[h] = mx;
            s_l[h] = sum;
        }
    }
    __syncthreads();

    // ---- phase 3: O = P.V on the tensor cores (mma.sync m16n8k16, fp32 accumulate) ----
    // A = P [head (8 of 16 rows) x 16 keys], encoded by attn_pack_p.  B = V [16 keys x 8 columns]: a B register holds
    // TWO KEYS of one column while V is key-major, so lane (g, t) loads D/8 contiguous elements (columns NJ g ..) of its
    // four keys 2t, 2t+1, 2t+8, 2t+9 and interleaves row pairs with PRMT; n-tile j column c stands for column
    // d = NJ c + j of V (a permutation of the columns, undone when the accumulators are written out).
    constexpr int NJ = D / 8;                 // n-tiles = V columns per lane and key row
    constexpr int NW = NJ / 2;                // 32-bit words of a lane's column chunk (2 elements each)
    constexpr bool kHalf = sizeof(T) == 2 && std::is_same<T, __half>::value;
    float* s_red = s_logit;                   // [warp][h][D], valid after the barrier below
    float o[NJ][4];
#pragma unroll
    for (int j = 0; j < NJ; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    for (int tile = warp; tile < ntiles; tile += kAttnWarps) {
        const int kb = tile * 16;
        uint32_t vw[4][NW];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int kk = kb + 2 * t + (r & 1) + (r >> 1) * 8;
#pragma unroll
            for (int w = 0; w < NW; ++w) vw[r][w] = 0u;
            if (kk < n) {
                const T* src = vbase + (size_t)(k0 + kk) * stride + g * NJ;
#pragma unroll
                for (int w4 = 0; w4 < NW / 4; ++w4) {
                    const uint4 v = ld_cg_u4(src + w4 * 8);
                    vw[r][w4 * 4 + 0] = v.x, vw[r][w4 * 4 + 1] = v.y, vw[r][w4 * 4 + 2] = v.z, vw[r][w4 * 4 + 3] = v.w;
                }
            }
        }
        uint32_t af[4] = {0u, 0u, 0u, 0u}, al[4] = {0u, 0u, 0u, 0u};
        if (g < mq) {
            const float* pr = s_logit + g * kAttnRowStride + kb + 2 * t;
            const float2 p0 = *reinterpret_cast<const float2*>(pr), p1 = *reinterpret_cast<const float2*>(pr + 8);
            const float q0 = kb + 2 * t < n ? p0.x : 0.f, q1 = kb + 2 * t + 1 < n ? p0.y : 0.f;
            const float q2 = kb + 2 * t + 8 < n ? p1.x : 0.f, q3 = kb + 2 * t + 9 < n ? p1.y : 0.f;
            attn_pack_p<T>(q0, q1, af[0], al[0]);
            attn_pack_p<T>(q2, q3, af[2], al[2]);
        }
#pragma unroll
        for (int w = 0; w < NW; ++w) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {            // element 2 w + e of the chunk = n-tile j
                const uint32_t sel = e ? 0x7632u : 0x5410u;
                const uint32_t b0 = __byte_perm(vw[0][w], vw[1][w], sel), b1 = __byte_perm(vw[2][w], vw[3][w], sel);
                mma_attn<T>(o[2 * w + e], af, b0, b1);
                if constexpr (!kHalf) mma_attn<T>(o[2 * w + e], al, b0, b1);
            }
        }
    }
    __syncthreads();   // everyone is done reading probabilities; reuse s_logit as the reduction buffer
    if (g < mq) {
        const float sc = kHalf ? (1.f / 1024.f) : 1.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            s_red[(warp * 8 + g) * D + NJ * (2 * t) + j] = o[j][0] * sc;
            s_red[(warp * 8 + g) * D + NJ * (2 * t + 1) + j] = o[j][1] * sc;
        }
    }
    __syncthreads();
    decode_attn_reduce_store<T, D>(cta, s_red, s_m, s_l, num_heads, num_splits, out, part_o, part_m, part_l);
}

}  // namespace zl

using namespace zl;

extern "C" size_t zl_decode_attention_workspace_bytes(int B, int len_q, int num_heads, int dim_head,
                                                      int max_len_buf) {
    if (B <= 0 || len_q <= 0 || num_heads <= 0 || dim_head <= 0) return 0;
    int splits = cdiv(max_len_buf > 0 ? max_len_buf : 1, kAttnMaxRange);
    if (splits < kAttnMaxSplits) splits = kAttnMaxSplits;
    return attn_parts_bytes((size_t)B * len_q * num_heads, splits, dim_head);
}

extern "C" int zl_decode_attention(const void* q, const int32_t* buf_lens, void* const* k_addrs,
                                   void* const* v_addrs, const int8_t* mask, float scale, int max_len_buf,
                                   void* out, int B, int len_q, int num_heads, int num_kv_heads, int dim_head,
                                   int bshd, void* workspace, size_t workspace_bytes, int dtype, int pdl,
                                   zl_stream_t stream) {
    ZL_CHECK_ARG(q && buf_lens && k_addrs && v_addrs && out && B > 0 && len_q > 0 && max_len_buf > 0);
    ZL_CHECK_ARG(num_heads > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0);
    ZL_CHECK_SUPPORTED(dim_head == 64 || dim_head == 128);
    ZL_CHECK_SUPPORTED(dtype == ZL_F16 || dtype == ZL_BF16);
    const int m_query = num_heads / num_kv_heads;
    int splits = attn_num_splits(B, len_q, num_kv_heads, m_query, max_len_buf);
    // latency regime: few CTAs of work -> 256-key splits on the warp-per-32-keys kernel (one __syncthreads per CTA)
    const int hgroups = (m_query + 7) / 8;
    const int short_splits = cdiv(max_len_buf, kShortRange);
    const bool use_short = short_splits <= kAttnMaxSplits &&
                           (long long)B * len_q * num_kv_heads * hgroups * short_splits <= 4 * device_sm_count();
    if (use_short) splits = short_splits;
    const size_t vheads = (size_t)B * len_q * num_heads;
    if (splits > 1) ZL_CHECK_ARG(workspace != nullptr && workspace_bytes >= attn_parts_bytes(vheads, splits, dim_head));
    const AttnParts part = attn_parts(workspace, vheads, splits, dim_head);
    dim3 grid(splits, num_kv_heads * hgroups, B * len_q), block(kAttnThreads);
#define ZL_ATTN_LAUNCH(TT, DD)                                                                                  \
    if (use_short) {                                                                                            \
        ZL_CHECK_CUDA(launch(k_decode_attn_warp<TT, DD>, grid, dim3(kWarpAttnWarps * 32),                       \
                             (size_t)warp_attn_smem_floats<DD>() * sizeof(float), stream, pdl != 0, (const TT*)q, \
                             buf_lens, (TT* const*)k_addrs, (TT* const*)v_addrs, mask, scale, (TT*)out, part.o, \
                             part.m, part.l, len_q, num_heads, num_kv_heads, m_query, splits, bshd));            \
    } else {                                                                                                    \
        ZL_CHECK_CUDA(launch(k_decode_attn<TT, DD>, grid, block, 0, stream, pdl != 0, (const TT*)q, buf_lens,   \
                             (TT* const*)k_addrs, (TT* const*)v_addrs, mask, scale, (TT*)out, part.o, part.m,   \
                             part.l, len_q, num_heads, num_kv_heads, m_query, splits, bshd));                   \
    }                                                                                                           \
    ZL_CHECK_CUDA(launch_attn_combine(part, vheads, DD, (TT*)out, splits, stream, pdl != 0));
    if (dtype == ZL_F16) {
        if (dim_head == 128) { ZL_ATTN_LAUNCH(__half, 128) } else { ZL_ATTN_LAUNCH(__half, 64) }
    } else {
        if (dim_head == 128) { ZL_ATTN_LAUNCH(__nv_bfloat16, 128) } else { ZL_ATTN_LAUNCH(__nv_bfloat16, 64) }
    }
#undef ZL_ATTN_LAUNCH
    return ZL_OK;
}
