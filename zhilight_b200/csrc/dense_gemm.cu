// Skinny dense GEMM y(M,N) = x(M,K) @ W(N,K)^T for M <= 32 per pass (lm_head, bf16/fp16 Linear at decode).
//
// Replaces the cuBLASLt GEMV the reference uses for unquantized Linear / lm_head at decode
// (src/nn/linear/linear.cpp:150-430 NormalLinear, src/nn/embedding/embedding.cu:353-392).
// HBM-bound: W is streamed once, straight from global memory into mma.sync A fragments
// (16-byte non-allocating loads, 4 k-steps in flight per warp); a k-permutation shared by the A and
// B fragments makes every load a contiguous 16 bytes (see DESIGN.md section 4.2).
#include "common.cuh"

extern unsigned long long* g_w4_trace;   // debug timeline buffer (zl_w4_set_trace), see w4a16_gemm_v3.cu

namespace zl {

constexpr int kDenseWarps = 8;
constexpr int kDenseUnroll = 4;   // k-steps (32 k each) in flight
// One CTA = kDenseWarps warps = (kDenseWarps / KS) row tiles of 16 weight rows, each split KS ways along K: small N
// (layer Linears of a 1B model: N/16 = 128 tiles) still puts >= 16 warps of loads in flight on every SM.

template <typename T>
__device__ __forceinline__ void mma_t(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma_t<__half>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    mma_16816_f16(d, a, b0, b1, d);
}
template <>
__device__ __forceinline__ void mma_t<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                                     uint32_t b1) {
    mma_16816_bf16(d, a, b0, b1, d);
}

// Persistent: a CTA walks tile groups blockIdx.x, blockIdx.x + gridDim.x, ... (lm_head: 8016 tiles on 296 CTAs) so that
// one wave of CTAs with UNROLL k-steps in flight per warp (>= 13 MB chip-wide) streams the whole matrix without the
// wave tails of a tile-per-warp grid.
template <typename T, typename TO, int NT, int KS, int UNROLL>
__global__ void __launch_bounds__(kDenseWarps * 32, 2)
k_dense_skinny(const T* __restrict__ x, int ldx, const T* __restrict__ w, const T* __restrict__ bias,
               TO* __restrict__ y, int mc, int N, int K, unsigned long long* trace) {
    constexpr int TPC = kDenseWarps / KS;   // tiles per CTA per pass
    __shared__ float red[KS > 1 ? kDenseWarps : 1][NT][4][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int ks = warp % KS;
    const int n_groups = (cdiv(N, 16) + TPC - 1) / TPC;
    // debug timeline: one record per launch, same format as the W4 kernels (trace[0] = launch counter, 16 words each);
    // CTA 0 stamps entry / wait_done / end, word 15 = 0xD marks a dense launch
    unsigned long long* tr = nullptr;
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) {
        tr = trace + 8 + (size_t)atomicAdd(trace, 1ull) * 16;
        tr[0] = globaltimer_ns();
        tr[15] = 0xDull;
    }
    pdl_trigger();
    const int all_steps = K / 32;
    const int s_lo = (int)((long long)all_steps * ks / KS), steps = (int)((long long)all_steps * (ks + 1) / KS);

    bool waited = false;
    for (int tg = blockIdx.x; tg < n_groups; tg += gridDim.x) {
        const int tile = tg * TPC + warp / KS;
        const int row0 = tile * 16;
        const bool live = row0 < N;
        const int ra = min(row0 + g, N - 1), rb = min(row0 + g + 8, N - 1);
        const T* wa = w + (size_t)ra * K + t * 8;
        const T* wb = w + (size_t)rb * K + t * 8;

        uint4 na[UNROLL], nb[UNROLL];
        if (live) {
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                if (s_lo + u < steps) {
                    na[u] = ld_nc_na_u4(wa + (size_t)(s_lo + u) * 32);
                    nb[u] = ld_nc_na_u4(wb + (size_t)(s_lo + u) * 32);
                }
            }
        }
        if (!waited) {   // the first weight loads are in flight before the predecessor kernel's results are needed
            pdl_wait();
            waited = true;
            if (tr) tr[1] = tr[2] = globaltimer_ns();
        }

        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[nt][c] = 0.f;

        for (int s0 = s_lo; live && s0 < steps; s0 += UNROLL) {
            uint4 xb[UNROLL][NT];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u)
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    const int tok = nt * 8 + g;
                    xb[u][nt] = (tok < mc && s0 + u < steps)
                                    ? ld_cg_u4(x + (size_t)tok * ldx + (size_t)(s0 + u) * 32 + t * 8)
                                    : make_uint4(0, 0, 0, 0);
                }
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                if (s0 + u < steps) {
                    const uint32_t a0[4] = {na[u].x, nb[u].x, na[u].y, nb[u].y};
                    const uint32_t a1[4] = {na[u].z, nb[u].z, na[u].w, nb[u].w};
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) {
                        mma_t<T>(acc[nt], a0, xb[u][nt].x, xb[u][nt].y);
                        mma_t<T>(acc[nt], a1, xb[u][nt].z, xb[u][nt].w);
                    }
                }
                // the registers just consumed take the load of the same slot one round ahead: UNROLL steps stay in flight
                const int sn = s0 + UNROLL + u;
                if (sn < steps) {
                    na[u] = ld_nc_na_u4(wa + (size_t)sn * 32);
                    nb[u] = ld_nc_na_u4(wb + (size_t)sn * 32);
                }
            }
        }

        if constexpr (KS > 1) {   // split-k partial sums meet in shared memory, added in k order
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                for (int c = 0; c < 4; ++c) red[warp][nt][c][lane] = acc[nt][c];
            __syncthreads();
            if (ks == 0) {
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        float sum = acc[nt][c];
#pragma unroll
                        for (int k2 = 1; k2 < KS; ++k2) sum += red[warp + k2][nt][c][lane];
                        acc[nt][c] = sum;
                    }
            }
            __syncthreads();   // red is reused by the next tile group
        }
        if (live && ks == 0) {
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int tok = nt * 8 + 2 * t + (c & 1);
                    const int row = row0 + g + ((c >> 1) ? 8 : 0);
                    if (tok < mc && row < N) {
                        float v = acc[nt][c];
                        if (bias) v += to_f32<T>(bias[row]);
                        y[(size_t)tok * N + row] = from_f32<TO>(v);
                    }
                }
            }
        }
    }
    if (!waited) pdl_wait();
    if (tr) tr[3] = globaltimer_ns();
    if (trace && threadIdx.x == 0) {   // last CTA to leave stamps the kernel's end (header words 4, 5)
        if (atomicAdd(&trace[4], 1ull) == gridDim.x - 1) {
            if (trace[5] == 0) trace[5] = globaltimer_ns();
            trace[4] = 0;
        }
    }
}

template <typename T, typename TO, int NT>
static cudaError_t launch_dense_ks(const T* x, int ldx, const T* w, const T* bias, TO* y, int mc, int N, int K,
                                   bool pdl, cudaStream_t stream) {
    const int tiles = cdiv(N, 16);
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    const int steps = K / 32;
    constexpr int UNROLL = NT == 1 ? 8 : 4;   // k-steps (2 x 16 B per lane each) in flight per warp
    const int slots = sms * 2 * kDenseWarps;  // resident warps: 2 CTAs per SM
    // split K over the warps of a CTA until the tiles fill the resident warps with little imbalance
    int ks = 1;
    while (ks < kDenseWarps && steps / (ks * 2) >= 2 * UNROLL &&
           (tiles * ks < slots || (tiles * ks) % slots > 0 && (tiles * ks) / slots < 4 && ks < 2))
        ks *= 2;
    dim3 block(kDenseWarps * 32);
#define ZL_DENSE_LAUNCH(KS_)                                                                                           \
    {                                                                                                                  \
        const int groups = cdiv(tiles, kDenseWarps / KS_);                                                             \
        const int grid = groups < sms * 2 ? groups : sms * 2;                                                          \
        return launch(k_dense_skinny<T, TO, NT, KS_, UNROLL>, dim3(grid), block, 0, stream, pdl, x, ldx, w, bias, y, mc, \
                      N, K, g_w4_trace);                                                                               \
    }
    if (ks == 1) ZL_DENSE_LAUNCH(1);
    if (ks == 2) ZL_DENSE_LAUNCH(2);
    if (ks == 4) ZL_DENSE_LAUNCH(4);
    ZL_DENSE_LAUNCH(8);
#undef ZL_DENSE_LAUNCH
}

template <typename T, typename TO>
static cudaError_t launch_dense(const T* x, int ldx, const T* w, const T* bias, TO* y, int mc, int N, int K,
                                bool pdl, cudaStream_t stream) {
    if (mc <= 8) return launch_dense_ks<T, TO, 1>(x, ldx, w, bias, y, mc, N, K, pdl, stream);
    if (mc <= 16) return launch_dense_ks<T, TO, 2>(x, ldx, w, bias, y, mc, N, K, pdl, stream);
    return launch_dense_ks<T, TO, 4>(x, ldx, w, bias, y, mc, N, K, pdl, stream);
}

template <typename T>
static cudaError_t dispatch_out(const T* x, int ldx, const T* w, const T* bias, void* y, int mc, int N, int K,
                                int out_dtype, bool pdl, cudaStream_t stream, size_t y_off) {
    if (out_dtype == ZL_F32)
        return launch_dense<T, float>(x, ldx, w, bias, static_cast<float*>(y) + y_off, mc, N, K, pdl, stream);
    return launch_dense<T, T>(x, ldx, w, bias, static_cast<T*>(y) + y_off, mc, N, K, pdl, stream);
}

}  // namespace zl

using namespace zl;

extern "C" int zl_dense_gemm_skinny(const void* x, int ldx, const void* w, const void* bias, void* y, int M,
                                    int N, int K, int dtype, int out_dtype, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(x && w && y && M > 0 && N > 0 && K > 0);
    ZL_CHECK_ARG(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_ARG(out_dtype == dtype || out_dtype == ZL_F32);
    ZL_CHECK_SUPPORTED(K % 32 == 0);
    ZL_CHECK_ARG(ldx >= K && ldx % 8 == 0);
    ZL_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0);
    for (int m0 = 0; m0 < M; m0 += 32) {
        const int mc = (M - m0) < 32 ? (M - m0) : 32;
        const bool use_pdl = pdl != 0 && m0 == 0;
        cudaError_t e;
        if (dtype == ZL_F16)
            e = dispatch_out<__half>(static_cast<const __half*>(x) + (size_t)m0 * ldx, ldx,
                                     static_cast<const __half*>(w), static_cast<const __half*>(bias), y, mc, N,
                                     K, out_dtype, use_pdl, stream, (size_t)m0 * N);
        else
            e = dispatch_out<__nv_bfloat16>(static_cast<const __nv_bfloat16*>(x) + (size_t)m0 * ldx, ldx,
                                            static_cast<const __nv_bfloat16*>(w),
                                            static_cast<const __nv_bfloat16*>(bias), y, mc, N, K, out_dtype,
                                            use_pdl, stream, (size_t)m0 * N);
        ZL_CHECK_CUDA(e);
    }
    return ZL_OK;
}
