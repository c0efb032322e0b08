// Latency-optimised decode attention for the small-batch regime (a batch-1 step has H_kv CTAs of work and sits
// between two GEMMs that each take a few microseconds): one WARP owns 32 keys of one kv-head group end to end --
// S = K.Q^T on the tensor cores, its own softmax statistics with shuffles only, P.V in fp32 -- so a CTA (<= 8 warps =
// 256 keys) has exactly ONE __syncthreads: the log-sum-exp merge of its warps.  Every global load of a warp (q, 32 K rows,
// 32 V rows) is issued before the first dependent instruction.
//
// Same mathematics as k_decode_attn / the reference (attention_kernel.cu:434-489, 674-725, 881-923): masked logits,
// fp32 exp, sum seeded with 1e-20, o = sum p.v in fp32; the per-warp partial results are merged with the reference's
// own split rule (KERNEL_mqa_combine), which is exact up to fp32 rounding.
#pragma once
#include "attn_common.cuh"

namespace zl {

constexpr int kWarpAttnWarps = 8;
constexpr int kWarpAttnRange = kWarpAttnWarps * 32;   // keys per CTA

template <int D>
constexpr int warp_attn_smem_floats() { return kWarpAttnWarps * (32 * 8 + 8 * D + 16); }   // per warp: P[32][8], o[8][D], m[8], l[8]

template <typename T, int D>
__global__ void __launch_bounds__(kWarpAttnWarps * 32)
k_decode_attn_warp(const T* __restrict__ q, const int32_t* __restrict__ buf_lens, T* const* __restrict__ k_addrs,
                   T* const* __restrict__ v_addrs, const int8_t* __restrict__ mask, float scale, T* __restrict__ out,
                   float* __restrict__ part_o, float* __restrict__ part_m, float* __restrict__ part_l, int len_q,
                   int num_heads, int num_kv_heads, int m_query, int num_splits, int bshd) {
    constexpr int NI = D / 32;
    constexpr int DC = D / 8;            // lanes covering one V row (16 bytes each)
    constexpr int RPI = 32 / DC;         // V rows per load instruction of the warp: 2 (D = 128) or 4 (D = 64)
    constexpr int VU = 32 / RPI;         // V loads per lane
    extern __shared__ __align__(16) float s_dyn[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    float* s_p = s_dyn + warp * (32 * 8 + 8 * D + 16);   // [key 32][head 8]
    float* s_o = s_p + 32 * 8;                           // [head 8][D]
    float* s_ml = s_o + 8 * D;                           // m[8], l[8]

    const DecodeAttnItem cta = decode_attn_prologue(buf_lens, len_q, m_query, num_splits);   // <= kWarpAttnRange keys
    const int mq = cta.mq;
    const int k0 = cta.k0 + warp * 32;               // this warp's keys [k0, k1)
    const int k1 = min(cta.k1, k0 + 32);
    const int n = max(0, k1 - k0);

    const size_t stride = bshd ? (size_t)num_kv_heads * D : (size_t)D;
    const size_t base = bshd ? (size_t)cta.hk * D : (size_t)cta.hk * cta.len_buf * D;
    const T* kbase = k_addrs[cta.b] + base;
    const T* vbase = v_addrs[cta.b] + base;
    const int8_t* mrow = cta.mask_row(mask, buf_lens, len_q);

    float m_w[2] = {-1e20f, -1e20f}, l_w[2] = {0.f, 0.f};   // heads 2t, 2t+1 of this lane
    float o[8][8];
#pragma unroll
    for (int h = 0; h < 8; ++h)
#pragma unroll
        for (int i = 0; i < 8; ++i) o[h][i] = 0.f;

    if (n > 0) {
        // ---- every load of the warp up front ----
        uint4 qf[NI], ka[2][NI], kb[2][NI];
        decode_attn_load_q<D>(qf, q, cta, num_heads, g, t);
#pragma unroll
        for (int tl = 0; tl < 2; ++tl) {
            const T* pa = kbase + (size_t)min(k0 + tl * 16 + g, k1 - 1) * stride + t * 8;
            const T* pb = kbase + (size_t)min(k0 + tl * 16 + g + 8, k1 - 1) * stride + t * 8;
#pragma unroll
            for (int i = 0; i < NI; ++i) {
                ka[tl][i] = ld_cg_u4(pa + i * 32);
                kb[tl][i] = ld_cg_u4(pb + i * 32);
            }
        }
        const int dc = lane % DC, sub = lane / DC;
        uint4 vv[VU];
        const T* vp = vbase + (size_t)k0 * stride + dc * 8;
#pragma unroll
        for (int u = 0; u < VU; ++u) {
            const int kk = sub + u * RPI;
            vv[u] = kk < n ? ld_cg_u4(vp + (size_t)kk * stride) : make_uint4(0, 0, 0, 0);
        }

        // ---- S = K.Q^T: lane (g,t) gets keys {g, g+8, 16+g, 24+g} x heads {2t, 2t+1} ----
        float sc[2][4];
#pragma unroll
        for (int tl = 0; tl < 2; ++tl) {
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < NI; ++i) {
                const uint32_t a0[4] = {ka[tl][i].x, kb[tl][i].x, ka[tl][i].y, kb[tl][i].y};
                const uint32_t a1[4] = {ka[tl][i].z, kb[tl][i].z, ka[tl][i].w, kb[tl][i].w};
                mma_attn<T>(acc, a0, qf[i].x, qf[i].y);
                mma_attn<T>(acc, a1, qf[i].z, qf[i].w);
            }
            const int ia = k0 + tl * 16 + g, ib = ia + 8;
            const bool va = ia < k1 && (!mrow || mrow[ia] != 0);
            const bool vb = ib < k1 && (!mrow || mrow[ib] != 0);
            sc[tl][0] = va ? acc[0] * scale : -INFINITY;   // (key ia, head 2t)
            sc[tl][1] = va ? acc[1] * scale : -INFINITY;   // (key ia, head 2t+1)
            sc[tl][2] = vb ? acc[2] * scale : -INFINITY;   // (key ib, head 2t)
            sc[tl][3] = vb ? acc[3] * scale : -INFINITY;
        }
        // ---- softmax statistics of the warp's 32 keys: reduce over g (lane bits 2..4) ----
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            float mx = fmaxf(fmaxf(sc[0][e], sc[0][e + 2]), fmaxf(sc[1][e], sc[1][e + 2]));
            mx = fmaxf(mx, -1e20f);
#pragma unroll
            for (int off = 4; off < 32; off <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            float sum = 0.f;
#pragma unroll
            for (int tl = 0; tl < 2; ++tl) {
                const float ea = expf(sc[tl][e] - mx), eb = expf(sc[tl][e + 2] - mx);
                sc[tl][e] = ea;
                sc[tl][e + 2] = eb;
                sum += ea + eb;
            }
#pragma unroll
            for (int off = 4; off < 32; off <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
            m_w[e] = mx;
            l_w[e] = sum;
        }
        // probabilities (unnormalised) to the warp's private smem tile
#pragma unroll
        for (int tl = 0; tl < 2; ++tl) {
            const int ra = tl * 16 + g, rb = ra + 8;
            *reinterpret_cast<float2*>(&s_p[ra * 8 + 2 * t]) = make_float2(sc[tl][0], sc[tl][1]);
            *reinterpret_cast<float2*>(&s_p[rb * 8 + 2 * t]) = make_float2(sc[tl][2], sc[tl][3]);
        }
        __syncwarp();
        // ---- O = P.V in fp32 from the registers loaded at the top ----
#pragma unroll
        for (int u = 0; u < VU; ++u) {
            const int kk = sub + u * RPI;
            if (kk < n) {
                float vf[8];
                unpack8<T>(vv[u], vf);
                const float4 p03 = *reinterpret_cast<const float4*>(&s_p[kk * 8]);
                const float4 p47 = *reinterpret_cast<const float4*>(&s_p[kk * 8 + 4]);
                const float pr[8] = {p03.x, p03.y, p03.z, p03.w, p47.x, p47.y, p47.z, p47.w};
#pragma unroll
                for (int h = 0; h < 8; ++h) {
                    if (h < mq) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) o[h][i] = fmaf(pr[h], vf[i], o[h][i]);
                    }
                }
            }
        }
#pragma unroll
        for (int h = 0; h < 8; ++h)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float v = o[h][i];
#pragma unroll
                for (int off = DC; off < 32; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
                o[h][i] = v;
            }
    }
    // ---- publish the warp's partial (m, l, o) ----
    if (g == 0) {   // lanes t = 0..3 hold the statistics of heads 2t, 2t+1
        s_ml[2 * t] = m_w[0];
        s_ml[2 * t + 1] = m_w[1];
        s_ml[8 + 2 * t] = l_w[0];
        s_ml[8 + 2 * t + 1] = l_w[1];
    }
    if (lane < DC) {
#pragma unroll
        for (int h = 0; h < 8; ++h)
            if (h < mq) {
                *reinterpret_cast<float4*>(&s_o[h * D + lane * 8]) = make_float4(o[h][0], o[h][1], o[h][2], o[h][3]);
                *reinterpret_cast<float4*>(&s_o[h * D + lane * 8 + 4]) = make_float4(o[h][4], o[h][5], o[h][6], o[h][7]);
            }
    }
    __syncthreads();
    // ---- merge the warps (KERNEL_mqa_combine rule) ----
    constexpr int WS = 32 * 8 + 8 * D + 16;
    for (int e = tid; e < mq * D; e += kWarpAttnWarps * 32) {
        const int h = e / D, d = e % D;
        float gm = -1e20f;
#pragma unroll
        for (int w = 0; w < kWarpAttnWarps; ++w) gm = fmaxf(gm, s_dyn[w * WS + 32 * 8 + 8 * D + h]);
        float gl = 1e-20f, acc = 0.f;
#pragma unroll
        for (int w = 0; w < kWarpAttnWarps; ++w) {
            const float f = expf(s_dyn[w * WS + 32 * 8 + 8 * D + h] - gm);
            gl += s_dyn[w * WS + 32 * 8 + 8 * D + 8 + h] * f;
            acc += s_dyn[w * WS + 32 * 8 + h * D + d] * f;
        }
        decode_attn_store<T, D>(cta, h, d, acc / gl, gm, gl, num_heads, num_splits, out, part_o, part_m, part_l);
    }
}

}  // namespace zl
