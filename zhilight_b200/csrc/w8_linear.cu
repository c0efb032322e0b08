// W8A8 Linear for decode-sized M: SmoothQuant INT8 (Int8Linear, src/nn/linear/linear.cpp:432-636) and
// per-tensor FP8 e4m3 (Fp8Linear, linear.cpp:1612-1695).
//
// The reference runs three launches per INT8 Linear -- quant_calc_scale (int8/quant_kernel.cu:15-47), an s32
// cuBLASLt GEMM with M padded to 32 (linear.cpp:591-616) and quant_scale_back (quant_kernel.cu:231-246) -- with an
// int32 (M,N) round trip through HBM, and three per FP8 Linear (segmented_max_reduction + T_KERNEL_cvt_half_fp8 +
// cuBLASLt fp8, fp8/fp8_util.cu:58-228).  Here: one activation-quant kernel (per token / per tensor, optionally
// fused with RMSNorm like layernorm_quant, quant_kernel.cu:106-227) and ONE GEMM kernel that streams the 8-bit
// weights once from HBM straight into mma.sync fragments (IMMA.16832 s8*s8->s32 / QMMA e4m3->f32) and applies the
// scale-back (+bias) in its epilogue.  HBM-bound: N*K bytes per call.
//
// Layout trick (same as dense_gemm.cu): the sum over k is order-free, so lane (g,t) loads 16 CONTIGUOUS bytes of
// weight row g (and g+8) per 64-k step and the activation fragment uses the same k permutation -- every global
// load is a full 16-byte vector, no shared-memory staging of the weights at all.
// Small N is covered by splitting K across the warps of a CTA (int32 partial sums add exactly).
//
// Block-scaled FP8 (BLK, QuantType 10 / Fp8Block, linear.cpp:1697-1960): each warp's K range is whole 128-k blocks,
// the 64-k steps of one block are steps 2 kb and 2 kb + 1 (the lane permutation stays inside a step), and after
// every block the QMMA sum is folded into an fp32 sum times sx[kb, token] * sw[row / 128, kb].
#include "common.cuh"

#include <cstdlib>

namespace zl {
// wgmma W8A8 kernel (w8_tc.cu)
bool w8_tc_supports(int N, int K);
template <typename T, bool FP8>
cudaError_t launch_w8_tc(const uint8_t* xq, const float* sx, const uint8_t* w, const void* sw, int sw_mode, const T* bias, T* y,
                         int mc, int N, int K, bool pdl, cudaStream_t stream, int sx_ld = 0);
}  // namespace zl

#include <cuda_fp8.h>

namespace zl {

constexpr int kW8Warps = 8;
constexpr int kW8Unroll = 4;    // 64-k steps in flight per warp (4 x 2 x 16 B per lane)

__device__ __forceinline__ void imma_s8s8(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void qmma_e4m3(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <bool FP8>
struct W8Acc {
    using type = int;
};
template <>
struct W8Acc<true> {
    using type = float;
};

// ---------------------------------------------------------------------------------------------
// activation quantisation
// ---------------------------------------------------------------------------------------------
template <typename V>
__device__ __forceinline__ V block_reduce(V v, V* sh, bool is_max) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = is_max ? warp_max(v) : warp_sum(v);
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    V r = sh[0];
    for (int i = 1; i < nw; ++i) r = is_max ? fmaxf(r, sh[i]) : r + sh[i];
    __syncthreads();
    return r;
}

// quant_calc_scale (quant_kernel.cu:15-47): scale = absmax/127, q = int8(nearbyint(x * (127/absmax))).
template <typename T>
__global__ void __launch_bounds__(256) k_int8_quant_per_token(const T* __restrict__ x, int ldx, int8_t* __restrict__ q,
                                                              float* __restrict__ scale, int K) {
    __shared__ float sh[8];
    pdl_trigger();
    pdl_wait();
    const T* row = x + (size_t)blockIdx.x * ldx;
    float amax = 0.f;
    for (int i = threadIdx.x * 8; i < K; i += blockDim.x * 8) {
        float v[8];
        unpack8<T>(ld_cg_u4(row + i), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[j]));
    }
    amax = block_reduce(amax, sh, true);
    const float bs = __fdiv_rn(127.f, amax);
    for (int i = threadIdx.x * 8; i < K; i += blockDim.x * 8) {
        float v[8];
        unpack8<T>(ld_cg_u4(row + i), v);
        uint32_t w[2] = {0, 0};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            // absmax == 0 gives 0 * inf = NaN, which the reference's float->int8 conversion turns into 0
            const float r = nearbyintf(__fmul_rn(v[j], bs));
            const int qi = (r == r) ? (int)r : 0;
            w[j >> 2] |= (uint32_t)(qi & 0xff) << (8 * (j & 3));
        }
        *reinterpret_cast<uint2*>(q + (size_t)blockIdx.x * K + i) = make_uint2(w[0], w[1]);
    }
    if (threadIdx.x == 0) scale[blockIdx.x] = __fdiv_rn(amax, 127.f);
}

// layernorm_quant (quant_kernel.cu:106-227): RMSNorm output in T plus its int8 twin.  The twin quantises
// v = x*w/scale (without rsqrt) and folds rsqrt into the scale; absmax is rounded through T (blockReduceMax<T>).
template <typename T>
__global__ void __launch_bounds__(256)
k_rmsnorm_quant(const T* __restrict__ x, const T* __restrict__ weight, T* __restrict__ y, int8_t* __restrict__ q,
                float* __restrict__ qscale, int D, float eps, float scale) {
    __shared__ float sh[8];
    pdl_trigger();
    pdl_wait();
    const T* row = x + (size_t)blockIdx.x * D;
    float sq = 0.f, amax = 0.f;
    for (int i = threadIdx.x * 8; i < D; i += blockDim.x * 8) {
        float v[8], w[8];
        unpack8<T>(ld_cg_u4(row + i), v);
        unpack8<T>(*reinterpret_cast<const uint4*>(weight + i), w);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sq = fmaf(v[j], v[j], sq);
            amax = fmaxf(amax, fabsf(__fmul_rn(v[j], w[j])));
        }
    }
    sq = block_reduce(sq, sh, false);
    amax = block_reduce(amax, sh, true);
    amax = to_f32<T>(from_f32<T>(amax));
    const float rs = rsqrtf(sq / (float)D + eps);
    const float bs = (float)(127.0 / (double)amax);
    for (int i = threadIdx.x * 8; i < D; i += blockDim.x * 8) {
        float v[8], w[8], o[8];
        unpack8<T>(ld_cg_u4(row + i), v);
        unpack8<T>(*reinterpret_cast<const uint4*>(weight + i), w);
        uint32_t qw[2] = {0, 0};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float vw = __fdiv_rn(__fmul_rn(v[j], w[j]), scale);
            o[j] = __fmul_rn(vw, rs);
            const float r = nearbyintf(__fmul_rn(vw, bs));
            const int qi = (r == r) ? (int)r : 0;
            qw[j >> 2] |= (uint32_t)(qi & 0xff) << (8 * (j & 3));
        }
        *reinterpret_cast<uint4*>(y + (size_t)blockIdx.x * D + i) = pack8<T>(o);
        *reinterpret_cast<uint2*>(q + (size_t)blockIdx.x * D + i) = make_uint2(qw[0], qw[1]);
    }
    if (threadIdx.x == 0) qscale[blockIdx.x] = (float)((double)__fmul_rn(amax, rs) / 127.);
}

// fp8 per-tensor dynamic quant (fp8_util.cu:110-228).  The reference's two launches (atomic absmax, convert)
// become one CTA-cooperative launch for decode-sized inputs: every CTA recomputes the (tiny) absmax itself, so
// there is no grid-wide dependency and no memset.
template <typename T>
__global__ void __launch_bounds__(256)
k_fp8_quant_per_tensor(const T* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ scale, size_t n) {
    __shared__ float sh[8];
    pdl_trigger();
    pdl_wait();
    float amax = 0.f;
    for (size_t i = (size_t)threadIdx.x * 8; i < n; i += (size_t)blockDim.x * 8) {
        float v[8];
        unpack8<T>(ld_cg_u4(x + i), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[j]));
    }
    amax = block_reduce(amax, sh, true);
    const float sc = __fdiv_rn(amax, 448.f);
    if (blockIdx.x == 0 && threadIdx.x == 0) *scale = sc;
    const float inv = __fdiv_rn(1.f, sc);
    for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; i < n; i += (size_t)gridDim.x * blockDim.x * 8) {
        float v[8];
        unpack8<T>(ld_cg_u4(x + i), v);
        uint32_t w[2] = {0, 0};
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            __half2 h2;
            if constexpr (std::is_same<T, __half>::value) {
                // fp16 input: the product is rounded in fp16 (__hmul2 with half(1/scale)), fp8_util.cu:77-80
                h2 = __hmul2(__floats2half2_rn(v[j], v[j + 1]), __float2half2_rn(inv));
            } else {
                h2 = __floats2half2_rn(__fmul_rn(inv, v[j]), __fmul_rn(inv, v[j + 1]));   // fp8_util.cu:74-76
            }
            const __nv_fp8x2_storage_t p = __nv_cvt_halfraw2_to_fp8x2(*reinterpret_cast<__half2_raw*>(&h2), __NV_SATFINITE, __NV_E4M3);
            w[j >> 2] |= (uint32_t)p << (16 * ((j >> 1) & 1));
        }
        *reinterpret_cast<uint2*>(q + i) = make_uint2(w[0], w[1]);
    }
}

// nn::fp8::per_token_cast_to_fp8 (fp8_util.cu:231-322): one warp per (token, 128-column group), 4 values per lane;
// amax clamped to 1e-4, q = e4m3(x * (448/amax)) with the fp32 product, scale = amax/448 stored column-major
// (K/128, scale_ld).  Each warp of a 256-thread CTA takes one group.
template <typename T>
__global__ void __launch_bounds__(256)
k_fp8_quant_per_token_group(const T* __restrict__ x, int ldx, uint8_t* __restrict__ q, float* __restrict__ scale,
                            int scale_ld, int M, int K) {
    pdl_trigger();
    pdl_wait();
    const int groups = K >> 7;
    const long long gi = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (gi >= (long long)M * groups) return;
    const int lane = threadIdx.x & 31;
    const int m = (int)(gi / groups), kb = (int)(gi % groups);
    const T* src = x + (size_t)m * ldx + kb * 128 + lane * 4;
    const uint2 raw = __ldcg(reinterpret_cast<const uint2*>(src));
    const T* h = reinterpret_cast<const T*>(&raw);
    float v[4];
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v[i] = to_f32<T>(h[i]);
        amax = fmaxf(amax, fabsf(v[i]));
    }
    amax = warp_max(amax);
    if (amax < 1e-4f) amax = 1e-4f;
    const float mul = __fdiv_rn(448.f, amax);
    uint32_t word = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __nv_fp8_storage_t c = __nv_cvt_float_to_fp8(__fmul_rn(v[i], mul), __NV_SATFINITE, __NV_E4M3);
        word |= (uint32_t)c << (8 * i);
    }
    *reinterpret_cast<uint32_t*>(q + (size_t)m * K + kb * 128 + lane * 4) = word;
    if (lane == 0) scale[(size_t)kb * scale_ld + m] = __fdiv_rn(amax, 448.f);
}

// quant_scale_back (quant_kernel.cu:231-246) for callers that still hold an int32 accumulator
template <typename T>
__global__ void k_int8_scale_back(const int32_t* __restrict__ acc, const float* __restrict__ sx, const void* __restrict__ sw,
                                  int sw_f32, T* __restrict__ y, int N) {
    const int r = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= N) return;
    const float s_w = sw_f32 ? static_cast<const float*>(sw)[c] : to_f32<T>(static_cast<const T*>(sw)[c]);
    y[(size_t)r * N + c] = from_f32<T>(__fmul_rn(__fmul_rn((float)acc[(size_t)r * N + c], sx[r]), s_w));
}

// ---------------------------------------------------------------------------------------------
// GEMM: y(M,N) = scale-back( xq(M,K) . wq(N,K)^T )
// ---------------------------------------------------------------------------------------------
// One CTA = kW8Warps warps = (kW8Warps / KS) row tiles of 16 weight rows, each split KS ways along K.
template <typename T, bool FP8, int NT, int KS, bool BLK>
__global__ void __launch_bounds__(kW8Warps * 32)
k_w8a8_skinny(const uint8_t* __restrict__ xq, const float* __restrict__ sx, const uint8_t* __restrict__ w,
              const void* __restrict__ sw, int sw_f32, const T* __restrict__ bias, T* __restrict__ y, int mc, int N,
              int K, int sx_ld) {
    static_assert(FP8 || !BLK, "block scales are fp8 only");
    using Acc = typename W8Acc<FP8>::type;
    constexpr int TPC = kW8Warps / KS;   // tiles per CTA
    __shared__ Acc red[KS > 1 ? kW8Warps : 1][NT][4][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int tile = blockIdx.x * TPC + warp / KS;
    const int ks = warp % KS;
    const int row0 = tile * 16;
    const bool live = row0 < N;
    pdl_trigger();

    const int steps = K / 64;
    // BLK: split by whole 128-k blocks, so s_lo is even and step s0 + u belongs to block (s0 + u) / 2 with parity u
    const int s_lo = BLK ? 2 * (int)((long long)(steps / 2) * ks / KS) : (int)((long long)steps * ks / KS);
    const int s_hi = BLK ? 2 * (int)((long long)(steps / 2) * (ks + 1) / KS) : (int)((long long)steps * (ks + 1) / KS);
    const int ra = min(row0 + g, N - 1), rb = min(row0 + g + 8, N - 1);
    const uint8_t* wa = w + (size_t)ra * K + t * 16;
    const uint8_t* wb = w + (size_t)rb * K + t * 16;

    uint4 na[kW8Unroll], nb[kW8Unroll];
    if (live) {
#pragma unroll
        for (int u = 0; u < kW8Unroll; ++u)
            if (s_lo + u < s_hi) {
                na[u] = ld_nc_na_u4(wa + (size_t)(s_lo + u) * 64);
                nb[u] = ld_nc_na_u4(wb + (size_t)(s_lo + u) * 64);
            }
    }
    pdl_wait();

    Acc acc[NT][4];
    float accb[BLK ? NT : 1][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[nt][c] = 0;
    if constexpr (BLK) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int c = 0; c < 4; ++c) accb[nt][c] = 0.f;
    }

    if (live) {
        for (int s0 = s_lo; s0 < s_hi; s0 += kW8Unroll) {
            uint4 ca[kW8Unroll], cb[kW8Unroll], xb[kW8Unroll][NT];
#pragma unroll
            for (int u = 0; u < kW8Unroll; ++u) {
                ca[u] = na[u];
                cb[u] = nb[u];
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    const int tok = nt * 8 + g;
                    xb[u][nt] = (tok < mc && s0 + u < s_hi) ? ld_cg_u4(xq + (size_t)tok * K + (size_t)(s0 + u) * 64 + t * 16)
                                                            : make_uint4(0, 0, 0, 0);
                }
            }
#pragma unroll
            for (int u = 0; u < kW8Unroll; ++u) {
                const int sn = s0 + kW8Unroll + u;
                if (sn < s_hi) {
                    na[u] = ld_nc_na_u4(wa + (size_t)sn * 64);
                    nb[u] = ld_nc_na_u4(wb + (size_t)sn * 64);
                }
            }
#pragma unroll
            for (int u = 0; u < kW8Unroll; ++u) {
                if (s0 + u < s_hi) {
                    const uint32_t a0[4] = {ca[u].x, cb[u].x, ca[u].y, cb[u].y};
                    const uint32_t a1[4] = {ca[u].z, cb[u].z, ca[u].w, cb[u].w};
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) {
                        if constexpr (FP8) {
                            qmma_e4m3(acc[nt], a0, xb[u][nt].x, xb[u][nt].y);
                            qmma_e4m3(acc[nt], a1, xb[u][nt].z, xb[u][nt].w);
                        } else {
                            imma_s8s8(acc[nt], a0, xb[u][nt].x, xb[u][nt].y);
                            imma_s8s8(acc[nt], a1, xb[u][nt].z, xb[u][nt].w);
                        }
                    }
                }
                if constexpr (BLK) {
                    if ((u & 1) && s0 + u < s_hi) {   // end of block kb: rows row0 .. row0 + 15 share one weight scale
                        const int kb = (s0 + u) >> 1;
                        const float s_w = static_cast<const float*>(sw)[(size_t)(row0 >> 7) * (K >> 7) + kb];
#pragma unroll
                        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int tok = nt * 8 + 2 * t + e;
                                const float s = tok < mc ? __ldg(sx + (size_t)kb * sx_ld + tok) * s_w : 0.f;
                                accb[nt][e] = fmaf(acc[nt][e], s, accb[nt][e]);
                                accb[nt][e + 2] = fmaf(acc[nt][e + 2], s, accb[nt][e + 2]);
                                acc[nt][e] = 0.f;
                                acc[nt][e + 2] = 0.f;
                            }
                    }
                }
            }
        }
    }
    if constexpr (BLK) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[nt][c] = accb[nt][c];
    }

    if constexpr (KS > 1) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int c = 0; c < 4; ++c) red[warp][nt][c][lane] = acc[nt][c];
        __syncthreads();
        if (ks != 0) return;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                Acc s = acc[nt][c];
#pragma unroll
                for (int k2 = 1; k2 < KS; ++k2) s += red[warp + k2][nt][c][lane];
                acc[nt][c] = s;
            }
    }
    if (!live) return;

#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int tok = nt * 8 + 2 * t + (c & 1);
            const int row = row0 + g + ((c >> 1) ? 8 : 0);
            if (tok < mc && row < N) {
                float v;
                if constexpr (BLK) {
                    v = acc[nt][c];   // scaled block by block above; Fp8Block has no bias
                } else if constexpr (FP8) {
                    // cuBLASLt fp8: D = (scaleA * scaleB) * acc (+ bias), functions::Gemm with A/B scales
                    // sw_f32 == 2: one scale per output row (several per-tensor-scaled projections fused along N)
                    const float s_w = sw_f32 == 2 ? static_cast<const float*>(sw)[row] : *static_cast<const float*>(sw);
                    v = acc[nt][c] * (sx[0] * s_w);
                    if (bias) v += to_f32<T>(bias[row]);
                } else {
                    // quant_scale_back (quant_kernel.cu:231-246): T(float(acc) * sx[m] * sw[n]) then add_bias in T
                    const float s_w = sw_f32 ? static_cast<const float*>(sw)[row] : to_f32<T>(static_cast<const T*>(sw)[row]);
                    v = __fmul_rn(__fmul_rn((float)acc[nt][c], sx[tok]), s_w);
                    if (bias) v = to_f32<T>(from_f32<T>(v)) + to_f32<T>(bias[row]);
                }
                y[(size_t)tok * N + row] = from_f32<T>(v);
            }
        }
    }
}

template <typename T, bool FP8, int NT, bool BLK>
static cudaError_t launch_w8_ks(const uint8_t* xq, const float* sx, const uint8_t* w, const void* sw, int sw_f32,
                                const T* bias, T* y, int mc, int N, int K, bool pdl, cudaStream_t st, int sx_ld) {
    const int tiles = cdiv(N, 16);
    // enough warps to keep ~13 MB of loads in flight chip-wide: aim for >= 16 warps per SM
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int steps = K / 64;
    int ks = 1;
    while (ks < kW8Warps && tiles * ks < sms * 16 && steps / (ks * 2) >= kW8Unroll) ks *= 2;
    if (BLK)   // every warp needs at least one whole 128-k block
        while (ks > 1 && (steps / 2) < ks) ks /= 2;
    dim3 block(kW8Warps * 32);
#define ZL_W8_LAUNCH(KS_)                                                                                          \
    return launch(k_w8a8_skinny<T, FP8, NT, KS_, BLK>, dim3(cdiv(tiles, kW8Warps / KS_)), block, 0, st, pdl, xq, sx, \
                  w, sw, sw_f32, bias, y, mc, N, K, sx_ld)
    if (ks == 1) ZL_W8_LAUNCH(1);
    if (ks == 2) ZL_W8_LAUNCH(2);
    if (ks == 4) ZL_W8_LAUNCH(4);
    ZL_W8_LAUNCH(8);
#undef ZL_W8_LAUNCH
}

template <typename T, bool FP8, bool BLK = false>
static cudaError_t launch_w8(const uint8_t* xq, const float* sx, const uint8_t* w, const void* sw, int sw_f32,
                             const T* bias, T* y, int mc, int N, int K, bool pdl, cudaStream_t st, int sx_ld = 0) {
    if (mc <= 8) return launch_w8_ks<T, FP8, 1, BLK>(xq, sx, w, sw, sw_f32, bias, y, mc, N, K, pdl, st, sx_ld);
    if (mc <= 16) return launch_w8_ks<T, FP8, 2, BLK>(xq, sx, w, sw, sw_f32, bias, y, mc, N, K, pdl, st, sx_ld);
    return launch_w8_ks<T, FP8, 4, BLK>(xq, sx, w, sw, sw_f32, bias, y, mc, N, K, pdl, st, sx_ld);
}

// Routing shared by zl_w8a8_gemm and zl_fp8_block_gemm.  With the reference's row-major (N, K) layout every 128-byte row
// segment of a TMA box comes from a different DRAM page, so at decode sizes the mma.sync kernel's 16-byte row-contiguous
// loads are used; the wgmma kernel takes over where the mma.sync kernel would re-stream the weights (M > 32: prefill
// chunks).  The crossover was not measured on H100.  tc(m0, mc, pdl) runs rows m0 .. m0 + mc - 1 (mc <= 256) on the
// wgmma kernel, skinny(m0, mc, pdl) on the mma.sync kernel (mc <= 32); only the first launch is PDL-launched.
template <typename TcFn, typename SkinnyFn>
static int w8_route(int M, int N, int K, int pdl, TcFn tc, SkinnyFn skinny) {
    static const int tc_min_m = getenv("ZL_W8_TC_MIN_M") ? atoi(getenv("ZL_W8_TC_MIN_M")) : 33;
    if (M >= tc_min_m && w8_tc_supports(N, K)) {
        static bool prepared[64] = {};   // zl_prepare() once per device: split-k workspace, opt-in shared memory
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64 || !prepared[dev]) {
            int rc = zl_prepare();
            if (rc != ZL_OK) return rc;
            if (dev >= 0 && dev < 64) prepared[dev] = true;
        }
        for (int m0 = 0; m0 < M; m0 += 256) {
            const int mc = (M - m0) < 256 ? (M - m0) : 256;
            ZL_CHECK_CUDA(tc(m0, mc, pdl != 0 && m0 == 0));
        }
        return ZL_OK;
    }
    for (int m0 = 0; m0 < M; m0 += 32) {
        const int mc = (M - m0) < 32 ? (M - m0) : 32;
        ZL_CHECK_CUDA(skinny(m0, mc, pdl != 0 && m0 == 0));
    }
    return ZL_OK;
}

}  // namespace zl

using namespace zl;

extern "C" int zl_int8_quant_per_token(const void* x, int ldx, void* q, float* scale, int M, int K, int dtype, int pdl,
                                       zl_stream_t stream) {
    ZL_CHECK_ARG(x && q && scale && M > 0 && K > 0);
    ZL_CHECK_ARG(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_SUPPORTED(K % 8 == 0 && ldx % 8 == 0 && ldx >= K);
    ZL_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 7) == 0);
    cudaError_t e;
    if (dtype == ZL_F16)
        e = launch(k_int8_quant_per_token<__half>, dim3(M), dim3(256), 0, stream, pdl != 0,
                   static_cast<const __half*>(x), ldx, static_cast<int8_t*>(q), scale, K);
    else
        e = launch(k_int8_quant_per_token<__nv_bfloat16>, dim3(M), dim3(256), 0, stream, pdl != 0,
                   static_cast<const __nv_bfloat16*>(x), ldx, static_cast<int8_t*>(q), scale, K);
    ZL_CHECK_CUDA(e);
    return ZL_OK;
}

extern "C" int zl_rmsnorm_quant(const void* x, const void* weight, void* y, void* q, float* qscale, int T_, int D,
                                float eps, float scale, int dtype, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(x && weight && y && q && qscale && T_ > 0 && D > 0);
    ZL_CHECK_ARG(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_SUPPORTED(D % 8 == 0);
    cudaError_t e;
    if (dtype == ZL_F16)
        e = launch(k_rmsnorm_quant<__half>, dim3(T_), dim3(256), 0, stream, pdl != 0, static_cast<const __half*>(x),
                   static_cast<const __half*>(weight), static_cast<__half*>(y), static_cast<int8_t*>(q), qscale, D, eps,
                   scale);
    else
        e = launch(k_rmsnorm_quant<__nv_bfloat16>, dim3(T_), dim3(256), 0, stream, pdl != 0,
                   static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(weight),
                   static_cast<__nv_bfloat16*>(y), static_cast<int8_t*>(q), qscale, D, eps, scale);
    ZL_CHECK_CUDA(e);
    return ZL_OK;
}

extern "C" int zl_fp8_quant_per_tensor(const void* x, void* q, float* scale, size_t n, int dtype, int pdl,
                                       zl_stream_t stream) {
    ZL_CHECK_ARG(x && q && scale && n > 0);
    ZL_CHECK_ARG(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_SUPPORTED(n % 8 == 0);
    // every CTA re-reads the whole input for the absmax: meant for decode-sized activations
    ZL_CHECK_SUPPORTED(n <= ((size_t)1 << 22));
    const int ctas = (int)((n / 8 + 255) / 256 < 64 ? (n / 8 + 255) / 256 : 64);
    cudaError_t e;
    if (dtype == ZL_F16)
        e = launch(k_fp8_quant_per_tensor<__half>, dim3(ctas), dim3(256), 0, stream, pdl != 0,
                   static_cast<const __half*>(x), static_cast<uint8_t*>(q), scale, n);
    else
        e = launch(k_fp8_quant_per_tensor<__nv_bfloat16>, dim3(ctas), dim3(256), 0, stream, pdl != 0,
                   static_cast<const __nv_bfloat16*>(x), static_cast<uint8_t*>(q), scale, n);
    ZL_CHECK_CUDA(e);
    return ZL_OK;
}

extern "C" int zl_int8_scale_back(const int32_t* acc, const float* x_scale, const void* w_scale, int w_scale_dtype,
                                  void* y, int M, int N, int dtype, zl_stream_t stream) {
    ZL_CHECK_ARG(acc && x_scale && w_scale && y && M > 0 && N > 0);
    ZL_CHECK_ARG(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_ARG(w_scale_dtype == ZL_F32 || w_scale_dtype == dtype);
    dim3 grid(cdiv(N, 256), M);
    if (dtype == ZL_F16)
        k_int8_scale_back<__half><<<grid, 256, 0, stream>>>(acc, x_scale, w_scale, w_scale_dtype == ZL_F32,
                                                            static_cast<__half*>(y), N);
    else
        k_int8_scale_back<__nv_bfloat16><<<grid, 256, 0, stream>>>(acc, x_scale, w_scale, w_scale_dtype == ZL_F32,
                                                                   static_cast<__nv_bfloat16*>(y), N);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_w8a8_gemm(const void* xq, const float* x_scale, const void* w, const void* w_scale,
                            int w_scale_dtype, const void* bias, void* y, int M, int N, int K, int kind, int dtype,
                            int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(xq && x_scale && w && w_scale && y && M > 0 && N > 0 && K > 0);
    ZL_CHECK_ARG(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_ARG(kind == ZL_W8_INT8 || kind == ZL_W8_FP8 || kind == ZL_W8_FP8_ROWS);
    ZL_CHECK_ARG(w_scale_dtype == ZL_F32 || w_scale_dtype == dtype);
    ZL_CHECK_ARG(kind == ZL_W8_INT8 || w_scale_dtype == ZL_F32);
    ZL_CHECK_SUPPORTED(K % 64 == 0);
    ZL_CHECK_ARG((reinterpret_cast<uintptr_t>(xq) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0);
    const uint8_t* xq8 = static_cast<const uint8_t*>(xq);
    const uint8_t* w8 = static_cast<const uint8_t*>(w);
    const int sw_f32 = kind == ZL_W8_FP8_ROWS ? 2 : (w_scale_dtype == ZL_F32 ? 1 : 0);
    const bool fp8 = kind != ZL_W8_INT8;
    const int sw_mode = fp8 ? (kind == ZL_W8_FP8_ROWS ? 2 : 3) : sw_f32;
    auto tc = [&](int m0, int mc, bool p) -> cudaError_t {
        // wgmma path (w8_tc.cu): both operands through the TMA engine, s32 / f32 register accumulators
        const float* sx = kind == ZL_W8_INT8 ? x_scale + m0 : x_scale;
        if (dtype == ZL_F16) {
            const __half* b = static_cast<const __half*>(bias);
            __half* yo = static_cast<__half*>(y) + (size_t)m0 * N;
            return fp8 ? launch_w8_tc<__half, true>(xq8 + (size_t)m0 * K, sx, w8, w_scale, sw_mode, b, yo, mc, N, K, p, stream)
                       : launch_w8_tc<__half, false>(xq8 + (size_t)m0 * K, sx, w8, w_scale, sw_mode, b, yo, mc, N, K, p, stream);
        }
        const __nv_bfloat16* b = static_cast<const __nv_bfloat16*>(bias);
        __nv_bfloat16* yo = static_cast<__nv_bfloat16*>(y) + (size_t)m0 * N;
        return fp8 ? launch_w8_tc<__nv_bfloat16, true>(xq8 + (size_t)m0 * K, sx, w8, w_scale, sw_mode, b, yo, mc, N, K, p, stream)
                   : launch_w8_tc<__nv_bfloat16, false>(xq8 + (size_t)m0 * K, sx, w8, w_scale, sw_mode, b, yo, mc, N, K, p, stream);
    };
    auto skinny = [&](int m0, int mc, bool p) -> cudaError_t {
        const float* sx = kind == ZL_W8_INT8 ? x_scale + m0 : x_scale;
#define ZL_W8_GO(TT, F8)                                                                                           \
    return launch_w8<TT, F8>(xq8 + (size_t)m0 * K, sx, w8, w_scale, sw_f32, static_cast<const TT*>(bias),           \
                             static_cast<TT*>(y) + (size_t)m0 * N, mc, N, K, p, stream)
        if (dtype == ZL_F16) {
            if (fp8) ZL_W8_GO(__half, true);
            ZL_W8_GO(__half, false);
        }
        if (fp8) ZL_W8_GO(__nv_bfloat16, true);
        ZL_W8_GO(__nv_bfloat16, false);
#undef ZL_W8_GO
    };
    return w8_route(M, N, K, pdl, tc, skinny);
}

extern "C" int zl_fp8_quant_per_token_group(const void* x, int ldx, void* q, float* scale, int scale_ld, int M, int K,
                                            int dtype, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(x && q && scale && M > 0 && K > 0 && ldx >= K && scale_ld >= M);
    ZL_CHECK_ARG(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_SUPPORTED(K % 128 == 0 && ldx % 4 == 0);
    ZL_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 7) == 0 && (reinterpret_cast<uintptr_t>(q) & 3) == 0);
    const long long groups = (long long)M * (K / 128);
    const dim3 grid((unsigned)((groups + 7) / 8));
    cudaError_t e;
    if (dtype == ZL_F16)
        e = launch(k_fp8_quant_per_token_group<__half>, grid, dim3(256), 0, stream, pdl != 0, static_cast<const __half*>(x),
                   ldx, static_cast<uint8_t*>(q), scale, scale_ld, M, K);
    else
        e = launch(k_fp8_quant_per_token_group<__nv_bfloat16>, grid, dim3(256), 0, stream, pdl != 0,
                   static_cast<const __nv_bfloat16*>(x), ldx, static_cast<uint8_t*>(q), scale, scale_ld, M, K);
    ZL_CHECK_CUDA(e);
    return ZL_OK;
}

extern "C" int zl_fp8_block_gemm(const void* xq, const float* x_scale, int x_scale_ld, const void* w, const float* w_scale,
                                 void* y, int M, int N, int K, int dtype, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(xq && x_scale && w && w_scale && y && M > 0 && N > 0 && K > 0 && x_scale_ld >= M);
    ZL_CHECK_ARG(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_SUPPORTED(K % 128 == 0);
    ZL_CHECK_ARG((reinterpret_cast<uintptr_t>(xq) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0);
    const uint8_t* xq8 = static_cast<const uint8_t*>(xq);
    const uint8_t* w8 = static_cast<const uint8_t*>(w);
    // routed like zl_w8a8_gemm; a chunk's x_scale is x_scale + m0 with the same leading dimension
    auto tc = [&](int m0, int mc, bool p) -> cudaError_t {
        if (dtype == ZL_F16)
            return launch_w8_tc<__half, true>(xq8 + (size_t)m0 * K, x_scale + m0, w8, w_scale, 4, nullptr,
                                              static_cast<__half*>(y) + (size_t)m0 * N, mc, N, K, p, stream, x_scale_ld);
        return launch_w8_tc<__nv_bfloat16, true>(xq8 + (size_t)m0 * K, x_scale + m0, w8, w_scale, 4, nullptr,
                                                 static_cast<__nv_bfloat16*>(y) + (size_t)m0 * N, mc, N, K, p, stream,
                                                 x_scale_ld);
    };
    auto skinny = [&](int m0, int mc, bool p) -> cudaError_t {
        if (dtype == ZL_F16)
            return launch_w8<__half, true, true>(xq8 + (size_t)m0 * K, x_scale + m0, w8, w_scale, 0, nullptr,
                                                 static_cast<__half*>(y) + (size_t)m0 * N, mc, N, K, p, stream, x_scale_ld);
        return launch_w8<__nv_bfloat16, true, true>(xq8 + (size_t)m0 * K, x_scale + m0, w8, w_scale, 0, nullptr,
                                                    static_cast<__nv_bfloat16*>(y) + (size_t)m0 * N, mc, N, K, p, stream,
                                                    x_scale_ld);
    };
    return w8_route(M, N, K, pdl, tc, skinny);
}
