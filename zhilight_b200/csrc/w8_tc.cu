// W8A8 Linear on the Hopper tensor cores: wgmma.mma_async s8 x s8 -> s32 (exact) and e4m3 x e4m3 -> f32 with register
// accumulators; BOTH operands arrive through the TMA engine (cp.async.bulk.tensor.2d, SWIZZLE_128B) straight from the
// reference's parameter layout and are read by wgmma from shared memory, so no CUDA-core instruction touches a weight byte.
//
// Replaces Int8Linear::forward = quant_calc_scale + cuBLASLt s32 GEMM (M padded to 32) + quant_scale_back
// (reference src/nn/linear/linear.cpp:560-636, src/nn/quant/int8/quant_kernel.cu:231-306) and Fp8Linear::forward's
// cuBLASLt fp8 GEMM (linear.cpp:1660-1695) for every M (decode and prefill chunks); the mma.sync kernel k_w8a8_skinny
// (w8_linear.cu) serves M <= 32 and K % 128 != 0 (w8_route).
//
// One CTA per SM, persistent over work items (128 weight rows x a k-slice); 9 warps:
//   warps 0-7  consumers : two warpgroups, warpgroup r owns weight rows 64 r .. 64 r + 63 of the tile and all NTOK tokens:
//                          4 x wgmma m64 x NTOK x 32 per stage, then scale-back (+bias), or split-k partials + last-CTA reduce
//   warp 8     producer  : per 128-byte k-stage one weight box (128 rows x 128 B) + one activation box (NTOK x 128 B)
// Block-scaled fp8 (BLK, QuantType 10): a 128-byte k-stage is one 128-wide scale block and a 128-row tile is one weight-scale
// row, so each stage's accumulator is folded into the fp32 sum times sx[kb, token] * sw[tile, kb].
// INT8 results are bit-identical to the reference's three-kernel path (s32 accumulation is exact in any order).
#include "common.cuh"
#include "tc_common.cuh"

#include <type_traits>

namespace zl {

constexpr int kW8TcThreads = 9 * 32;
constexpr int kW8WarpProducer = 8;

template <int NTOK>
struct W8TcCfg {
    static constexpr int kAStage = kTcRows * 128;
    static constexpr int kXStage = NTOK * 128;
    static constexpr int ST = NTOK <= 32 ? 8 : (NTOK <= 64 ? 7 : (NTOK <= 128 ? 6 : 4));
    static constexpr int kAOff = 0;
    static constexpr int kXOff = ST * kAStage;
    static constexpr int kBarOff = kXOff + ST * kXStage;
    static constexpr int kNumBars = 2 * ST;          // full[ST], empty[ST]
    static constexpr int kMiscOff = kBarOff + kNumBars * 8;
    static constexpr int kBytes = kMiscOff + 16 + 1024;
    static_assert(kBytes <= 232448, "shared memory");
};

struct alignas(64) W8TcParams {
    CUtensorMap wmap;          // w (N, K) 8-bit row-major, box {128 B, 128 rows}
    CUtensorMap xmap;          // xq (M, K) 8-bit row-major, box {128 B, NTOK rows}
    const float* sx;           // int8: (M) per-token scales; fp8: one scale; block: (K/128, sx_ld) column-major
    const void* sw;            // int8: (N) f32 or T; fp8: one f32 or (N) f32 rows; block: (ceil(N/128), K/128) f32
    int sw_mode;               // 0: T per row, 1: f32 per row, 2: f32 per row (fp8 rows), 3: one f32 (fp8), 4: block
    int sx_ld;
    const void* bias;
    void* y;
    int M, N, K, S;
    float* ws;
    unsigned* counters;
    unsigned* err;
};

// one output element: acc is the s32 sum (int8) or the f32 sum (fp8)
template <typename T, bool FP8, bool BLK>
__device__ __forceinline__ void w8_epilogue1(const W8TcParams& p, int row, int tok, float acc) {
    if (row >= p.N || tok >= p.M) return;
    if constexpr (BLK) {   // the block scales were applied per k-stage; no bias (Fp8Block has none)
        static_cast<T*>(p.y)[(size_t)tok * p.N + row] = from_f32<T>(acc);
        return;
    }
    const T* bias = static_cast<const T*>(p.bias);
    float s_w;
    if (p.sw_mode == 0) s_w = to_f32<T>(static_cast<const T*>(p.sw)[row]);
    else if (p.sw_mode == 3) s_w = *static_cast<const float*>(p.sw);
    else s_w = static_cast<const float*>(p.sw)[row];
    float r;
    if constexpr (FP8) {
        r = acc * (p.sx[0] * s_w);                       // cuBLASLt fp8: D = (scaleA * scaleB) * acc (+ bias)
        if (bias) r += to_f32<T>(bias[row]);
    } else {
        // quant_scale_back (quant_kernel.cu:231-246): T(float(acc) * sx[m] * sw[n]), then add_bias in T
        r = __fmul_rn(__fmul_rn(acc, p.sx[tok]), s_w);
        if (bias) r = to_f32<T>(from_f32<T>(r)) + to_f32<T>(bias[row]);
    }
    static_cast<T*>(p.y)[(size_t)tok * p.N + row] = from_f32<T>(r);
}

template <typename T, bool FP8, int NTOK, bool BLK>
__global__ void __launch_bounds__(kW8TcThreads, 1) k_w8a8_tc(const __grid_constant__ W8TcParams p) {
    static_assert(FP8 || !BLK, "block scales are fp8 only");
    using C = W8TcCfg<NTOK>;
    using Acc = typename std::conditional<FP8, float, int>::type;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::kBarOff);
    uint64_t* empty = full + C::ST;
    uint32_t* s_last = reinterpret_cast<uint32_t*>(smem + C::kMiscOff);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int KS = p.K / 128;                      // 128-byte k-stages
    const int n_tiles = (p.N + kTcRows - 1) / kTcRows, S = p.S;
    const int n_items = n_tiles * S;

    if (threadIdx.x == 0) {
        for (int i = 0; i < C::ST; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 8);             // one arrival per consumer warp
        }
        mbar_fence_init();
    }
    pdl_trigger();
    __syncthreads();

    if (warp == kW8WarpProducer) {
        if (lane == 0) {
            int st = 0;
            uint32_t ph = 0;
            bool waited = false;
            for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
                const int tile = it / S, split = it % S;
                const int s0 = (split * KS) / S, s1 = ((split + 1) * KS) / S;
                for (int ks = s0; ks < s1; ++ks) {
                    mbar_wait_wd(&empty[st], ph ^ 1u, p.err, 0x1100 + st);
                    mbar_expect_tx(&full[st], C::kAStage + C::kXStage);
                    // weights are constants: their boxes may be requested before the predecessor kernel has finished
                    tma_load_2d(smem + C::kAOff + st * C::kAStage, &p.wmap, ks * 128, tile * kTcRows, &full[st]);
                    if (!waited) {
                        pdl_wait();   // the quantised activations come from the predecessor kernel
                        waited = true;
                    }
                    tma_load_2d(smem + C::kXOff + st * C::kXStage, &p.xmap, ks * 128, 0, &full[st]);
                    if (++st == C::ST) {
                        st = 0;
                        ph ^= 1u;
                    }
                }
            }
        }
        return;
    }

    // ---------------- consumers: warpgroup wr, rows 64 wr + 16 (warp % 4) + g (+ 8) of the tile ----------------
    const int wr = warp >> 2, g = lane >> 2, tig = lane & 3;
    const int m0 = wr * 64 + (warp & 3) * 16 + g;   // rows m0 and m0 + 8; tokens 8 j + 2 tig + e
    const int ct = threadIdx.x;                     // 0 .. 255
    pdl_wait();
    int st = 0;
    uint32_t ph = 0;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const int tile = it / S, split = it % S;
        const int s0 = (split * KS) / S, s1 = ((split + 1) * KS) / S;
        Acc acc[NTOK / 2];
        // fp8: wgmma accumulates e4m3 products with less than fp32 precision, so each 128-byte k-stage starts a fresh
        // accumulator that is then added into an fp32 one (int8 sums are exact and accumulate in place)
        float accf[FP8 ? NTOK / 2 : 1];
        if constexpr (FP8) {
#pragma unroll
            for (int i = 0; i < NTOK / 2; ++i) accf[i] = 0.f;
        }
        for (int ks = s0; ks < s1; ++ks) {
            mbar_wait_wd(&full[st], ph, p.err, 0x1400 + st);
            const uint64_t ad = wg_desc_sw128(smem_u32(smem + C::kAOff + st * C::kAStage + wr * 64 * 128));
            const uint64_t xd = wg_desc_sw128(smem_u32(smem + C::kXOff + st * C::kXStage));
            wg_fence();
#pragma unroll
            for (int k32 = 0; k32 < 4; ++k32) {   // 32 bytes along K per wgmma inside the 128-byte swizzle atom
                const uint32_t accum = ((!FP8 && ks > s0) || k32 > 0) ? 1u : 0u;
                if constexpr (FP8) wg_e4m3_ss<NTOK>(acc, ad + (uint64_t)(k32 * 2), xd + (uint64_t)(k32 * 2), accum);
                else wg_s8_ss<NTOK>(acc, ad + (uint64_t)(k32 * 2), xd + (uint64_t)(k32 * 2), accum);
            }
            wg_commit();
            if constexpr (BLK) {
                // one weight scale for the tile, one x scale per token; the weight scale loads while the wgmmas run
                const float s_w = static_cast<const float*>(p.sw)[(size_t)tile * KS + ks];
                const float* sxk = p.sx + (size_t)ks * p.sx_ld;
                wg_wait_all();
#pragma unroll
                for (int j = 0; j < NTOK / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int tok = 8 * j + 2 * tig + e;
                        const float sc = tok < p.M ? __ldg(sxk + tok) * s_w : 0.f;
                        accf[4 * j + e] = fmaf(acc[4 * j + e], sc, accf[4 * j + e]);
                        accf[4 * j + e + 2] = fmaf(acc[4 * j + e + 2], sc, accf[4 * j + e + 2]);
                    }
            } else {
                wg_wait_all();
                if constexpr (FP8) {
#pragma unroll
                    for (int i = 0; i < NTOK / 2; ++i) accf[i] += acc[i];
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
            if (++st == C::ST) {
                st = 0;
                ph ^= 1u;
            }
        }
        if (S == 1) {
#pragma unroll
            for (int j = 0; j < NTOK / 8; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    w8_epilogue1<T, FP8, BLK>(p, tile * kTcRows + m0 + (e >> 1) * 8, 8 * j + 2 * tig + (e & 1),
                                        FP8 ? (float)accf[FP8 ? 4 * j + e : 0] : (float)acc[4 * j + e]);
            continue;
        }
        float* wsp = p.ws + ((size_t)(tile * S + split) * p.M) * kTcRows;
#pragma unroll
        for (int j = 0; j < NTOK / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int tok = 8 * j + 2 * tig + (e & 1);
                float v;
                if constexpr (FP8) v = accf[4 * j + e];
                else v = __int_as_float(acc[4 * j + e]);
                if (tok < p.M) __stcg(wsp + (size_t)tok * kTcRows + m0 + (e >> 1) * 8, v);
            }
        __threadfence();
        consumer_bar();
        if (ct == 0) *s_last = (atomicAdd(&p.counters[tile], 1u) == (unsigned)(S - 1)) ? 1u : 0u;
        consumer_bar();
        const bool last = *s_last != 0u;
        consumer_bar();
        if (last) {
            // the last arriver adds the k-slices in split order (deterministic) and runs the epilogue
            __threadfence();
            const float* base = p.ws + ((size_t)tile * S * p.M) * kTcRows;
#pragma unroll 1
            for (int idx = ct; idx < p.M * kTcRows; idx += 256) {
                const int tok = idx / kTcRows, m = idx % kTcRows;
                float v;
                if constexpr (FP8) {
                    v = 0.f;
                    for (int s = 0; s < S; ++s) v += __ldcg(base + (size_t)s * p.M * kTcRows + idx);
                } else {
                    int a = 0;
                    for (int s = 0; s < S; ++s) a += __float_as_int(__ldcg(base + (size_t)s * p.M * kTcRows + idx));
                    v = (float)a;
                }
                w8_epilogue1<T, FP8, BLK>(p, tile * kTcRows + m, tok, v);
            }
            if (ct == 0) p.counters[tile] = 0u;
        }
    }
}

// k-split so that short-and-wide GEMMs still fill the SMs; >= 8 stages of 128 bytes per item
static int w8_pick_splits(int n_tiles, int KS, int mc, size_t ws_bytes) {
    const int sms = device_sm_count();
    int best = 1;
    float best_score = -1.f;
    for (int s = 1; s <= 8 && s * 8 <= KS; ++s) {
        const long long items = (long long)n_tiles * s;
        if (s > 1 && (size_t)items * mc * kTcRows * 4 > ws_bytes) break;
        const long long waves = (items + sms - 1) / sms;
        const float score = (float)items / (float)(waves * sms) - 0.03f * (s - 1);
        if (score > best_score + 1e-6f) {
            best_score = score;
            best = s;
        }
    }
    return best;
}

bool w8_tc_supports(int N, int K) {
    return K % 128 == 0 && N >= 1 && (N + kTcRows - 1) / kTcRows <= kTcMaxTiles;
}

template <typename T, bool FP8, int NTOK, bool BLK>
static cudaError_t launch_w8_tc_t(const W8TcParams& q, dim3 grid, bool pdl, cudaStream_t stream) {
    return launch(k_w8a8_tc<T, FP8, NTOK, BLK>, grid, dim3(kW8TcThreads), (size_t)W8TcCfg<NTOK>::kBytes, stream, pdl, q);
}

// mc <= 256 rows of one pass (fp8: passes of <= 128 rows, its promoted accumulators take twice the registers).
// sw_mode 4 (block scales, FP8 only): sx is (K/128, sx_ld) column-major, sw (ceil(N/128), K/128) row-major.
// zl_prepare() must have run on this device (split-k workspace, opt-in shared memory).
template <typename T, bool FP8>
cudaError_t launch_w8_tc(const uint8_t* xq, const float* sx, const uint8_t* w, const void* sw, int sw_mode, const T* bias, T* y,
                         int mc, int N, int K, bool pdl, cudaStream_t stream, int sx_ld) {
    TcDeviceState* st = tc_state();
    if (!st || !st->ws) return cudaErrorNotSupported;
    const bool blk = sw_mode == 4;
    if (blk && !FP8) return cudaErrorInvalidValue;
    if (FP8 && mc > 128) {
        for (int r0 = 0; r0 < mc; r0 += 128) {   // per-tensor: one scale for all tokens, only x and y move
            const int rows = mc - r0 < 128 ? mc - r0 : 128;
            const cudaError_t e = launch_w8_tc<T, FP8>(xq + (size_t)r0 * K, blk ? sx + r0 : sx, w, sw, sw_mode, bias,
                                                       y + (size_t)r0 * N, rows, N, K, pdl, stream, sx_ld);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    const int ntok = mc <= 32 ? 32 : mc <= 64 ? 64 : mc <= 128 ? 128 : 256;
    W8TcParams q;
    if (!tc_make_map_2d(&q.wmap, w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, (uint64_t)N, (uint64_t)K, (uint64_t)K, kTcRows) ||
        !tc_make_map_2d(&q.xmap, xq, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, (uint64_t)mc, (uint64_t)K, (uint64_t)K, (uint32_t)ntok))
        return cudaErrorInvalidValue;
    q.sx = sx;
    q.sw = sw;
    q.sw_mode = sw_mode;
    q.sx_ld = sx_ld;
    q.bias = bias;
    q.y = y;
    q.M = mc;
    q.N = N;
    q.K = K;
    const int n_tiles = (N + kTcRows - 1) / kTcRows;
    q.S = w8_pick_splits(n_tiles, K / 128, mc, st->ws_bytes);
    q.ws = st->ws;
    q.counters = st->counters;
    q.err = st->err;
    const int items = n_tiles * q.S, sms = device_sm_count();
    const dim3 grid(items < sms ? items : sms);
    if constexpr (FP8) {
        if (blk) {
            switch (ntok) {
                case 32: return launch_w8_tc_t<T, true, 32, true>(q, grid, pdl, stream);
                case 64: return launch_w8_tc_t<T, true, 64, true>(q, grid, pdl, stream);
                case 128: return launch_w8_tc_t<T, true, 128, true>(q, grid, pdl, stream);
                default: return cudaErrorInvalidValue;
            }
        }
    }
    switch (ntok) {
        case 32: return launch_w8_tc_t<T, FP8, 32, false>(q, grid, pdl, stream);
        case 64: return launch_w8_tc_t<T, FP8, 64, false>(q, grid, pdl, stream);
        case 128: return launch_w8_tc_t<T, FP8, 128, false>(q, grid, pdl, stream);
        default:
            if constexpr (FP8) return cudaErrorInvalidValue;
            else return launch_w8_tc_t<T, FP8, 256, false>(q, grid, pdl, stream);
    }
}

template cudaError_t launch_w8_tc<__half, false>(const uint8_t*, const float*, const uint8_t*, const void*, int, const __half*,
                                                 __half*, int, int, int, bool, cudaStream_t, int);
template cudaError_t launch_w8_tc<__half, true>(const uint8_t*, const float*, const uint8_t*, const void*, int, const __half*,
                                                __half*, int, int, int, bool, cudaStream_t, int);
template cudaError_t launch_w8_tc<__nv_bfloat16, false>(const uint8_t*, const float*, const uint8_t*, const void*, int,
                                                        const __nv_bfloat16*, __nv_bfloat16*, int, int, int, bool, cudaStream_t, int);
template cudaError_t launch_w8_tc<__nv_bfloat16, true>(const uint8_t*, const float*, const uint8_t*, const void*, int,
                                                       const __nv_bfloat16*, __nv_bfloat16*, int, int, int, bool, cudaStream_t, int);

// opt-in shared-memory sizes must be set outside stream capture: called from zl_prepare
cudaError_t prepare_w8_tc() {
    cudaError_t e;
#define ZL_W8TC_SET(TT, F8, NT, B)                                                                                  \
    if ((e = cudaFuncSetAttribute(k_w8a8_tc<TT, F8, NT, B>, cudaFuncAttributeMaxDynamicSharedMemorySize,            \
                                  W8TcCfg<NT>::kBytes)) != cudaSuccess)                                            \
        return e;
#define ZL_W8TC_ALL(TT, F8, B) ZL_W8TC_SET(TT, F8, 32, B) ZL_W8TC_SET(TT, F8, 64, B) ZL_W8TC_SET(TT, F8, 128, B)
    ZL_W8TC_ALL(__half, false, false) ZL_W8TC_ALL(__half, true, false) ZL_W8TC_ALL(__nv_bfloat16, false, false)
    ZL_W8TC_ALL(__nv_bfloat16, true, false) ZL_W8TC_ALL(__half, true, true) ZL_W8TC_ALL(__nv_bfloat16, true, true)
    ZL_W8TC_SET(__half, false, 256, false) ZL_W8TC_SET(__nv_bfloat16, false, 256, false)
#undef ZL_W8TC_ALL
#undef ZL_W8TC_SET
    return cudaSuccess;
}

}  // namespace zl
