// W4A16 skinny GEMM, persistent + pipelined variant (the default), with optional fused prologue/epilogues:
//   prologue : RMSNorm of the input row (nn::LayerNorm, layernorm.cu:9-42) folded in -- x*w_ln feeds the MMA,
//              sum(x^2) is accumulated from the same registers, rsqrt(mean+eps) scales the accumulators;
//   epilogues: bias, SwiGLU (gemm_fuse_gate_in / gate_mul_inplace), residual add (element_add_scale),
//              qkv split + RoPE + KV append (rope_qk_cache + copy_to_rag_buffer2).
//
// Differences to the first variant (w4a16_gemm.cu), all aimed at keeping the HBM stream continuous:
//   * grid = min(#super-tiles, 2 per SM); each CTA walks super-tiles blockIdx.x, +gridDim.x, ... and every
//     warp's 4-stage bulk-TMA ring runs ACROSS tile boundaries, so the next tile's weights are in flight while
//     the current tile is reduced and written out (v1 CTAs each did one load -> wait -> compute round trip);
//   * the split-k reduction buffer is separate from the ring (double-buffered for M <= 8: one __syncthreads
//     per tile);
//   * 2 CTAs per SM leave room for the next kernel's CTAs to become resident under programmatic dependent
//     launch and pre-fill their rings.
#include "common.cuh"
#include "w4_layout.cuh"
#include "w4_params.h"

namespace zl {

// Two shapes of CTA (picked per GEMM by the number of 32-row super-tiles):
//   wide  : 8 warps, 5-stage rings, 2 CTAs/SM, persistent over tiles        (N/32 > #SMs: qkv, gate/up)
//   tall  : 16 warps, 4-stage rings, 1 CTA/SM, k split 16 ways              (N/32 <= #SMs: o_proj, down)
// Either way ~140-170 KB of weights are in flight per SM, which is what it takes to cover the ~2 us loaded
// HBM latency at 6.5 TB/s (Little's law: 13 MB chip-wide).
template <int NT, int WARPS, int STAGES>
struct V2Smem {
    static constexpr int kRingBytes = WARPS * STAGES * kW4BlockBytes;
    static constexpr int kRedBufs = (NT == 1 && WARPS == 8) ? 2 : 1;
    static constexpr int kRedFloats = WARPS * NT * 8 * 32;
    static constexpr int kBarOff = kRingBytes;
    static constexpr int kRedOff = kBarOff + WARPS * STAGES * 8;
    static constexpr int kSsOff = kRedOff + kRedBufs * kRedFloats * 4;          // [warps][NT*8] sum of squares
    static constexpr int kRstdOff = kSsOff + WARPS * NT * 8 * 4;                // [NT*8]
    static constexpr int kXOff = (kRstdOff + NT * 8 * 4 + 127) & ~127;          // optional x cache [mc][K + 32] halves
    static constexpr int kBytes = kXOff;
};
// (dynamic smem budgets)
// largest dynamic smem that still lets two CTAs share an SM (227 KB usable, 1 KB reserved per CTA) / one CTA
constexpr int kV2TwoCtaBudget = 115000;
constexpr int kV2OneCtaBudget = 231000;
__host__ __device__ inline int x_row_bytes(int K) { return K * 2 + 64; }   // +64 B: conflict-free LDS.128 across tokens

template <int NT, bool NORM>
__device__ __forceinline__ void load_bfrag_v2(uint4 (&b)[NT][4], const W4Params& p, int kbase, int g, int t,
                                              float (&ss)[NT]) {
    uint4 wl[4];
    if (NORM) {
#pragma unroll
        for (int ii = 0; ii < 4; ++ii)
            wl[ii] = *reinterpret_cast<const uint4*>(p.ln_w + kbase + ii * 32 + t * 8);
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const int tok = nt * 8 + g;
        if (tok < p.mc) {
            const __half* src = p.x + (size_t)tok * p.ldx + kbase + t * 8;
#pragma unroll
            for (int ii = 0; ii < 4; ++ii) {
                uint4 v = ld_cg_u4(src + ii * 32);
                if (NORM) {
                    __half2* hv = reinterpret_cast<__half2*>(&v);
                    const __half2* hw = reinterpret_cast<const __half2*>(&wl[ii]);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 f = __half22float2(hv[e]);
                        ss[nt] = fmaf(f.x, f.x, ss[nt]);
                        ss[nt] = fmaf(f.y, f.y, ss[nt]);
                        hv[e] = __hmul2(hv[e], hw[e]);
                    }
                }
                b[nt][ii] = v;
            }
        } else {
#pragma unroll
            for (int ii = 0; ii < 4; ++ii) b[nt][ii] = make_uint4(0, 0, 0, 0);
        }
    }
}

template <int NT, bool NORM, bool XC, int WARPS, int STAGES>
__global__ void __launch_bounds__(WARPS * 32, ((NT <= 2 && WARPS == 8) ? 2 : 1)) k_w4a16_v2(const W4Params p) {
    using S = V2Smem<NT, WARPS, STAGES>;
    constexpr int kV2Warps = WARPS;
    constexpr int kV2Stages = STAGES;
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int G = p.K / kW4GroupK;
    const int g_begin = (warp * G) / kV2Warps;
    const int g_end = ((warp + 1) * G) / kV2Warps;
    const int ng = g_end - g_begin;
    const int n_tiles = p.N / 32;
    const int my_tiles = (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total = my_tiles * ng;   // ring items of this warp

    uint8_t* ring = smem + warp * (kV2Stages * kW4BlockBytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kBarOff) + warp * kV2Stages;
    float* red = reinterpret_cast<float*>(smem + S::kRedOff);
    float* s_ss = reinterpret_cast<float*>(smem + S::kSsOff);
    float* s_rstd = reinterpret_cast<float*>(smem + S::kRstdOff);

    auto item_src = [&](int it) -> const uint8_t* {
        const int tile = (int)blockIdx.x + (it / ng) * (int)gridDim.x;
        const int gi = g_begin + it % ng;
        return p.packed + ((size_t)tile * G + gi) * kW4BlockBytes;
    };

    pdl_trigger();
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < kV2Stages; ++s) mbar_init(&bars[s], 1);
        mbar_fence_init();
#pragma unroll
        for (int s = 0; s < kV2Stages; ++s) {
            if (s < total) {
                mbar_expect_tx(&bars[s], kW4BlockBytes);
                bulk_g2s(ring + s * kW4BlockBytes, item_src(s), kW4BlockBytes, &bars[s]);
            }
        }
    }
    __syncwarp();
    pdl_wait();   // weights above are constants; x / residual / KV below come from predecessor kernels

    // ---- optional: stage x (times the RMSNorm weight) in shared memory once per CTA ----
    uint8_t* xs = smem + S::kXOff;
    const int xrow = x_row_bytes(p.K);
    if (XC) {
        const int chunks = p.K / 8;   // 16-byte chunks per token row
        for (int tok = 0; tok < p.mc; ++tok) {
            float sq = 0.f;
            for (int ch = threadIdx.x; ch < chunks; ch += blockDim.x) {
                uint4 v = ld_cg_u4(p.x + (size_t)tok * p.ldx + ch * 8);
                if (NORM) {
                    const uint4 wv = *reinterpret_cast<const uint4*>(p.ln_w + ch * 8);
                    __half2* hv = reinterpret_cast<__half2*>(&v);
                    const __half2* hw = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 f = __half22float2(hv[e]);
                        sq = fmaf(f.x, f.x, sq);
                        sq = fmaf(f.y, f.y, sq);
                        hv[e] = __hmul2(hv[e], hw[e]);
                    }
                }
                *reinterpret_cast<uint4*>(xs + (size_t)tok * xrow + ch * 16) = v;
            }
            if (NORM) {
                sq = warp_sum(sq);
                if (lane == 0) s_ss[warp * (NT * 8) + tok] = sq;
            }
        }
        __syncthreads();
        if (NORM) {
            if (threadIdx.x < p.mc) {
                float v = 0.f;
#pragma unroll
                for (int w = 0; w < kV2Warps; ++w) v += s_ss[w * (NT * 8) + threadIdx.x];
                s_rstd[threadIdx.x] = rsqrtf(v / (float)p.K + p.eps);
            }
            __syncthreads();
        }
    }

    const __half2 one16 = __half2half2(__ushort_as_half((unsigned short)0x2c00));   // 1/16
    const float zero4[4] = {0.f, 0.f, 0.f, 0.f};
    float ss[NT];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) ss[nt] = 0.f;

    int it = 0;
    for (int ti = 0; ti < my_tiles; ++ti) {
        const int st = (int)blockIdx.x + ti * (int)gridDim.x;
        float acc[2][NT][4];
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < NT; ++b)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;

        float ss_dummy[NT];
        for (int i = 0; i < ng; ++i, ++it) {
            const int s = it % kV2Stages;
            const uint32_t parity = (uint32_t)(it / kV2Stages) & 1u;
            uint4 bcur[NT][4];
            if (XC) {
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    const int tok = nt * 8 + g;
                    if (tok < p.mc) {
                        const uint8_t* src = xs + (size_t)tok * xrow + ((g_begin + i) * kW4GroupK + t * 8) * 2;
#pragma unroll
                        for (int ii = 0; ii < 4; ++ii) bcur[nt][ii] = *reinterpret_cast<const uint4*>(src + ii * 64);
                    } else {
#pragma unroll
                        for (int ii = 0; ii < 4; ++ii) bcur[nt][ii] = make_uint4(0, 0, 0, 0);
                    }
                }
            } else if (NORM && ti == 0) {
                // sum(x^2) only needs one pass over K: take it from the first tile
                load_bfrag_v2<NT, NORM>(bcur, p, (g_begin + i) * kW4GroupK, g, t, ss);
            } else {
                load_bfrag_v2<NT, NORM>(bcur, p, (g_begin + i) * kW4GroupK, g, t, ss_dummy);
            }

            mbar_wait(&bars[s], parity);
            const uint8_t* blk = ring + s * kW4BlockBytes;
            if (p.dbg & 1) {   // stream probe: touch one word so the copy cannot be elided, skip the math
                acc[0][0][0] += __uint_as_float(*reinterpret_cast<const uint32_t*>(blk + lane * 4)) * 1e-30f;
            } else
#pragma unroll
            for (int tt = 0; tt < 2; ++tt) {
                const __half2 sc = *reinterpret_cast<const __half2*>(blk + kW4ScaleOff + (tt * 8 + g) * 4);
                const uint32_t zz = blk[kW4ZeroOff + tt * 8 + g];
                const __half2 z1 = __half2half2(__ushort_as_half((unsigned short)(0xe400u | (zz & 0xFu))));
                const __half2 z16 = __half2half2(__ushort_as_half((unsigned short)(0xd400u | (zz & 0xF0u))));
                float accg[NT][4];
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const uint4 wv = *reinterpret_cast<const uint4*>(blk + ((tt * 2 + hh) * 32 + lane) * 16);
                    const uint32_t wj[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int j = hh * 4 + jj;
                        uint32_t w = wj[jj];
                        uint32_t a[4];
                        uint32_t p0 = lop3_and_or<0x000f000fu, 0x64006400u>(w);
                        uint32_t p1 = lop3_and_or<0x00f000f0u, 0x64006400u>(w);
                        w >>= 8;
                        uint32_t p2 = lop3_and_or<0x000f000fu, 0x64006400u>(w);
                        uint32_t p3 = lop3_and_or<0x00f000f0u, 0x64006400u>(w);
                        __half2 h0 = __hadd2(*reinterpret_cast<__half2*>(&p0), z1);
                        __half2 h1 = __hfma2(*reinterpret_cast<__half2*>(&p1), one16, z16);
                        __half2 h2 = __hadd2(*reinterpret_cast<__half2*>(&p2), z1);
                        __half2 h3 = __hfma2(*reinterpret_cast<__half2*>(&p3), one16, z16);
                        a[0] = *reinterpret_cast<uint32_t*>(&h0);
                        a[1] = *reinterpret_cast<uint32_t*>(&h1);
                        a[2] = *reinterpret_cast<uint32_t*>(&h2);
                        a[3] = *reinterpret_cast<uint32_t*>(&h3);
#pragma unroll
                        for (int nt = 0; nt < NT; ++nt) {
                            const uint4 bv = bcur[nt][j >> 1];
                            const uint32_t b0 = (j & 1) ? bv.z : bv.x;
                            const uint32_t b1 = (j & 1) ? bv.w : bv.y;
                            if (j == 0)
                                mma_16816_f16(accg[nt], a, b0, b1, zero4);
                            else
                                mma_16816_f16(accg[nt], a, b0, b1, accg[nt]);
                        }
                    }
                }
                const float s_lo = __low2float(sc), s_hi = __high2float(sc);
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    acc[tt][nt][0] = fmaf(s_lo, accg[nt][0], acc[tt][nt][0]);
                    acc[tt][nt][1] = fmaf(s_lo, accg[nt][1], acc[tt][nt][1]);
                    acc[tt][nt][2] = fmaf(s_hi, accg[nt][2], acc[tt][nt][2]);
                    acc[tt][nt][3] = fmaf(s_hi, accg[nt][3], acc[tt][nt][3]);
                }
            }
            __syncwarp();   // every lane is done reading ring slot s
            if (lane == 0 && it + kV2Stages < total) {
                mbar_expect_tx(&bars[s], kW4BlockBytes);
                bulk_g2s(ring + s * kW4BlockBytes, item_src(it + kV2Stages), kW4BlockBytes, &bars[s]);
            }
        }

        // ---- split-k reduction across the warps ----
        float* myred = red + (S::kRedBufs == 2 ? (ti & 1) * S::kRedFloats : 0) + warp * (NT * 8 * 32);
#pragma unroll
        for (int tt = 0; tt < 2; ++tt)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const int tok = nt * 8 + 2 * t;
                const int row = tt * 16 + g;
                myred[tok * 32 + row] = acc[tt][nt][0];
                myred[(tok + 1) * 32 + row] = acc[tt][nt][1];
                myred[tok * 32 + row + 8] = acc[tt][nt][2];
                myred[(tok + 1) * 32 + row + 8] = acc[tt][nt][3];
            }
        if (NORM && !XC && ti == 0) {
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                float v = ss[nt];
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                if (t == 0) s_ss[warp * (NT * 8) + nt * 8 + g] = v;
            }
        }
        __syncthreads();
        if (NORM && !XC && ti == 0) {
            if (threadIdx.x < NT * 8) {
                float v = 0.f;
#pragma unroll
                for (int w = 0; w < kV2Warps; ++w) v += s_ss[w * (NT * 8) + threadIdx.x];
                s_rstd[threadIdx.x] = rsqrtf(v / (float)p.K + p.eps);
            }
            __syncthreads();
        }

        const float* rbase = red + (S::kRedBufs == 2 ? (ti & 1) * S::kRedFloats : 0);
        auto sum_red = [&](int idx) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < kV2Warps; ++w) v += rbase[w * (NT * 8 * 32) + idx];
            return v;
        };
        const int n0 = st * 32;
        if (p.epi == ZL_EPI_SWIGLU) {
            const int n_out = p.N / 2;
            for (int e = threadIdx.x; e < p.mc * 16; e += blockDim.x) {
                const int tok = e >> 4, oc = e & 15;
                const int rg = (oc >> 3) * 16 + (oc & 7);   // gate row; the matching up row is rg + 8
                float gate = sum_red(tok * 32 + rg);
                float up = sum_red(tok * 32 + rg + 8);
                if (NORM) {
                    gate *= s_rstd[tok];
                    up *= s_rstd[tok];
                }
                if (p.bias) {
                    gate += __half2float(p.bias[n0 + rg]);
                    up += __half2float(p.bias[n0 + rg + 8]);
                }
                const float gr = __half2float(__float2half_rn(gate));
                const float ur = __half2float(__float2half_rn(up));
                p.y[(size_t)tok * n_out + st * 16 + oc] = __float2half_rn(silu_f(gr) * ur);
            }
        } else if (p.epi == ZL_EPI_QKV_ROPE) {
            // packed rows: 16-row tile = 8 rows c followed by their RoPE partners c + d/2 (zl_qkv_rope_row_map)
            const int d = p.dim_head, half_dim = d / 2;
            const int tiles_per_head = d / 32;
            const int head = st / tiles_per_head, jt = st % tiles_per_head;
            for (int e = threadIdx.x; e < p.mc * 16; e += blockDim.x) {
                const int tok = e >> 4, oc = e & 15;
                const int rlo = (oc >> 3) * 16 + (oc & 7);
                const int c = jt * 16 + oc;                 // column within the head, c < d/2
                float lo = sum_red(tok * 32 + rlo), hi = sum_red(tok * 32 + rlo + 8);
                if (NORM) {
                    lo *= s_rstd[tok];
                    hi *= s_rstd[tok];
                }
                if (p.bias) {
                    lo += __half2float(p.bias[n0 + rlo]);
                    hi += __half2float(p.bias[n0 + rlo + 8]);
                }
                // the reference materialises the fused qkv GEMV output in fp16 before rope_qk_cache
                lo = __half2float(__float2half_rn(lo));
                hi = __half2float(__float2half_rn(hi));
                __half olo, ohi;
                const bool is_v = head >= p.num_heads + p.num_kv_heads;
                if (is_v) {
                    olo = __float2half_rn(lo);
                    ohi = __float2half_rn(hi);
                } else {
                    const float* cs = p.cos + (size_t)tok * d;
                    const float* sn = p.sin + (size_t)tok * d;
                    olo = __float2half_rn(lo * cs[c] - hi * sn[c]);                       // rope_common.cuh:22-23
                    ohi = __float2half_rn(hi * cs[c + half_dim] + lo * sn[c + half_dim]);  // rope_common.cuh:24-25
                }
                if (head < p.num_heads) {
                    __half* dst = p.q_out + ((size_t)tok * p.num_heads + head) * d;
                    dst[c] = olo;
                    dst[c + half_dim] = ohi;
                } else {
                    const int pl = p.placement[tok];
                    if (pl >= 0) {
                        const bool is_k = !is_v;
                        const int hk = is_k ? head - p.num_heads : head - p.num_heads - p.num_kv_heads;
                        __half* base = (is_k ? p.k_addrs : p.v_addrs)[p.token_batch[tok]];
                        __half* dst = base + ((size_t)pl * p.num_kv_heads + hk) * d;      // BSHD
                        dst[c] = olo;
                        dst[c + half_dim] = ohi;
                    }
                }
            }
        } else {
            for (int e = threadIdx.x; e < p.mc * 32; e += blockDim.x) {
                const int tok = e >> 5, row = e & 31;
                float v = sum_red(tok * 32 + row);
                if (NORM) v *= s_rstd[tok];
                if (p.bias) v += __half2float(p.bias[n0 + row]);
                __half h = __float2half_rn(v);
                if (p.epi == ZL_EPI_RESIDUAL)
                    h = __float2half_rn(__half2float(h) + __half2float(p.residual[(size_t)tok * p.N + n0 + row]));
                p.y[(size_t)tok * p.N + n0 + row] = h;
            }
        }
        if (S::kRedBufs == 1) __syncthreads();   // single reduction buffer: readers must finish before the next tile
    }
}

// The kernels of one ring shape, by fused RMSNorm prologue and by staging x in shared memory (XC).  NT token tiles of 8:
// 16 warps (tall: one CTA per SM, k split 16 ways) for NT <= 2, 8 warps (two CTAs per SM) otherwise.
using V2Kernel = void (*)(W4Params);
struct V2Variant {
    int nt, warps, ring_bytes;   // ring_bytes: shared memory without the staged x
    V2Kernel k[2][2];            // [NORM][XC]
};
template <int NT, int W, int ST>
static V2Variant v2_variant() {
    return {NT, W, V2Smem<NT, W, ST>::kBytes,
            {{k_w4a16_v2<NT, false, false, W, ST>, k_w4a16_v2<NT, false, true, W, ST>},
             {k_w4a16_v2<NT, true, false, W, ST>, k_w4a16_v2<NT, true, true, W, ST>}}};
}
// Every v2 kernel: launch_w4_v2 runs one of these and prepare_w4_v2 opts all of them in
static const V2Variant kV2Variants[] = {v2_variant<1, 8, 5>(), v2_variant<2, 8, 4>(), v2_variant<4, 8, 4>(),
                                        v2_variant<1, 16, 4>(), v2_variant<2, 16, 4>()};
static int v2_budget(const V2Variant& v) { return v.warps == 8 ? kV2TwoCtaBudget : kV2OneCtaBudget; }

cudaError_t launch_w4_v2(const W4Params& p, bool pdl, cudaStream_t stream) {
    const int sms = device_sm_count();
    const int nt = p.mc <= 8 ? 1 : p.mc <= 16 ? 2 : 4;
    const bool tall = nt <= 2 && p.N / 32 <= sms && p.K / kW4GroupK >= 32;
    for (const V2Variant& v : kV2Variants) {
        if (v.nt != nt || v.warps != (tall ? 16 : 8)) continue;
        // stage x in shared memory when the CTA budget allows (always true for M = 1 at the Llama shapes)
        const int x_bytes = p.mc * x_row_bytes(p.K);
        const bool xc = v.ring_bytes + x_bytes <= v2_budget(v);
        const int tiles = p.N / 32, max_ctas = sms * (v.warps == 8 ? 2 : 1);
        return launch(v.k[p.ln_w != nullptr][xc], dim3(tiles < max_ctas ? tiles : max_ctas), dim3(v.warps * 32),
                      (size_t)(v.ring_bytes + (xc ? x_bytes : 0)), stream, pdl, p);
    }
    return cudaErrorNotSupported;
}

cudaError_t prepare_w4_v2() {
    for (const V2Variant& v : kV2Variants)
        for (const auto& by_xc : v.k)
            for (int xc = 0; xc < 2; ++xc) {
                const cudaError_t e = cudaFuncSetAttribute(by_xc[xc], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                           xc ? v2_budget(v) : v.ring_bytes);
                if (e != cudaSuccess) return e;
            }
    return cudaSuccess;
}

}  // namespace zl
