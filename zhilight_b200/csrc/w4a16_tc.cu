// W4A16 GEMM on the Hopper tensor cores: wgmma.mma_async (f16 x f16 -> f32) with the dequantised weights as the A operand
// in REGISTERS, activations through tensor-TMA as the shared-memory B operand, register accumulators.  Serves every M the
// exact-integer mma.sync kernel (w4a16_gemm_v3.cu) cannot stage: batch 17..256 decode and chunked prefill.
//
// Replaces the reference's Marlin kernel (src/nn/quant/marlin/gptq_marlin.cu:425-1620), the M <= 40 GEMV tiles of
// KERNEL_gemm_warp_reduce (src/nn/quant/gptq/q_gemm_k_major.cu:176-237, 580-686: the weight matrix is streamed
// ceil(M/16) times) and the M > 40 route "dequantise the whole matrix to fp16 in HBM, then cuBLASLt"
// (q_gemm_k_major.cu:843-905, 1083-1100).  Same arithmetic contract as that route: w = (q - z) * s rounded to fp16
// once, fp16 x fp16 products, fp32 accumulation over all of K.
//
// One CTA per SM.  The work is the list of (128-row tile, 128-k group) units in tile-major order, cut into one contiguous
// range per CTA ("stream-k"): a tile that lies inside one range is finished by that CTA alone, a tile cut by a range
// boundary is shared by the CTAs that own its pieces -- each writes its fp32 partial tile to a per-CTA slot as tagged words,
// the owners then split the tile's tokens among themselves and add the pieces in k order (deterministic).  Every CTA does
// its (at most two) partial pieces FIRST, so the exchange overlaps the full tiles that follow.
//
//   warps 0-7  consumers : two warpgroups; warpgroup r owns weight rows 64 r .. 64 r + 63 of the tile (two ZLW4I 32-row
//                          blocks).  Per 128-k group each thread converts its A fragments (rows g and g + 8 of its warp's
//                          16-row slab: PRMT 0x64xx / 0x54xx magic, exact q - z, one HMUL2 by the group scale), issues
//                          8 x wgmma m64 x NTOK x 16, and at the end of a piece runs the bias / residual / SwiGLU /
//                          qkv-RoPE-KV epilogue from its accumulators
//   warp 8     producer  : tensor-TMA (4-D / 3-D maps) of the 4 ZLW4I records of a stage and of the x tile
//                          (box 64 k x NTOK tokens, SWIZZLE_128B, OOB rows = 0)
//
// A ZLW4I word holds 4 k of row g (low nibbles) and of row g + 8 (high nibbles), which is exactly the row pair of a wgmma
// A fragment: one 16-bit half of a word gives a thread both rows for its two consecutive k.  The 8 row groups g of a warp
// read 16-byte chunks 64 B apart -- a 4-way bank conflict in the plain record layout -- so the nibble words arrive through a
// tensor map with 64-byte swizzle (chunk ^= (row >> 1) & 3): conflict-free, the HBM format is unchanged.  The 80-byte
// scale / zero trailers of the four records of a stage come through a second (unswizzled) map.
#include "common.cuh"
#include "w4_layout.cuh"
#include "w4_params.h"
#include "tc_common.cuh"

#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>

namespace zl {

struct alignas(64) W4TcParams {
    CUtensorMap xmap;           // x (M, K) fp16 row-major, box {64, NTOK}, 128-byte swizzle
    CUtensorMap wmap;           // ZLW4I nibble words as [N/32][G][32 rows][64 B], box {64 B, 32, 1, 4}, 64-byte swizzle
    CUtensorMap tmap;           // the 80-byte scale / zero trailers as [N/32][G][80 B], box {80 B, 1, 4}
    const uint8_t* packed;      // ZLW4I
    const __half* bias;         // indexed by PACKED row
    const __half* residual;
    __half* y;
    int M, N, K, epi;
    uint2* ws;                  // [2 * CTA + slot][M][128] tagged words {fp32 partial sum, tag}: all zero between launches
    unsigned* err;              // watchdog code
    const float* cos;
    const float* sin;
    __half* q_out;
    const int32_t* token_batch;
    const int32_t* placement;
    __half* const* k_addrs;
    __half* const* v_addrs;
    int num_heads, num_kv_heads, dim_head;
};

// ---- epilogue of one token for one row pair -----------------------------------------------------------------------------
// Packed rows blk * 32 + 16 tt + g (lo) and + 8 (hi) are partners (gate / up, RoPE low / high half); a wgmma accumulator
// fragment holds both for the same token.
__device__ __forceinline__ float tc_silu(float x) { return __fdividef(x, 1.0f + __expf(-x)); }

__device__ __forceinline__ void tc_epilogue_pair(const W4TcParams& p, int blk, int tt, int g, int tok, float vlo, float vhi) {
    if (tok >= p.M) return;
    const int plo = blk * 32 + tt * 16 + g, phi = plo + 8;
    const float lo = __half2float(__float2half_rn(vlo + (p.bias ? __half2float(p.bias[plo]) : 0.f)));
    const float hi = __half2float(__float2half_rn(vhi + (p.bias ? __half2float(p.bias[phi]) : 0.f)));
    if (p.epi == ZL_EPI_SWIGLU) {
        p.y[(size_t)tok * (p.N / 2) + blk * 16 + tt * 8 + g] = __float2half_rn(tc_silu(lo) * hi);
    } else if (p.epi == ZL_EPI_QKV_ROPE) {
        const int d = p.dim_head, half_dim = d / 2, tiles_per_head = d / 32;
        const int head = blk / tiles_per_head, jt = blk % tiles_per_head;
        const int c = jt * 16 + tt * 8 + g;
        const bool is_v = head >= p.num_heads + p.num_kv_heads;
        __half olo, ohi;
        if (is_v) {
            olo = __float2half_rn(lo);
            ohi = __float2half_rn(hi);
        } else {
            const float* cs = p.cos + (size_t)tok * d;
            const float* sn = p.sin + (size_t)tok * d;
            olo = __float2half_rn(lo * cs[c] - hi * sn[c]);
            ohi = __float2half_rn(hi * cs[c + half_dim] + lo * sn[c + half_dim]);
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
                __half* dst = base + ((size_t)pl * p.num_kv_heads + hk) * d;
                dst[c] = olo;
                dst[c + half_dim] = ohi;
            }
        }
    } else {
        __half hlo = __float2half_rn(lo), hhi = __float2half_rn(hi);
        if (p.epi == ZL_EPI_RESIDUAL) {
            hlo = __float2half_rn(lo + __half2float(p.residual[(size_t)tok * p.N + plo]));
            hhi = __float2half_rn(hi + __half2float(p.residual[(size_t)tok * p.N + phi]));
        }
        p.y[(size_t)tok * p.N + plo] = hlo;
        p.y[(size_t)tok * p.N + phi] = hhi;
    }
}

template <int NTOK>
struct TsCfg {
    static constexpr int kThreads = 9 * 32;                             // 2 consumer warpgroups + 1 producer warp
    static constexpr int kWarpProducer = 8;
    static constexpr int ST = NTOK <= 64 ? 8 : (NTOK <= 128 ? 5 : 3);   // stages of one 128-k group
    static constexpr int kXGroup = 2 * NTOK * 128;                      // [k atom (64 k)][token][128 B]
    static constexpr int kNibGroup = 4 * 2048, kTrGroup = 384;          // 4 x 80 B trailers, padded to the TMA alignment
    static constexpr int kXOff = 0;
    static constexpr int kNibOff = kXOff + ST * kXGroup;
    static constexpr int kTrOff = kNibOff + ST * kNibGroup;
    static constexpr int kBarOff = kTrOff + ST * kTrGroup;
    static constexpr int kNumBars = 2 * ST;
    static constexpr int kBytes = kBarOff + kNumBars * 8 + 1024;        // + slack for the manual 1024-byte alignment
    static_assert(kBytes <= 232448, "shared memory");
};

// ---- stream-k schedule ------------------------------------------------------------------------------------------------
// U = n_tiles * G units in tile-major order; CTA b owns [b U / P, (b + 1) U / P).  Its pieces, in processing order: the one
// at the start of the range, the one at its end (both possibly partial tiles), then the whole tiles in between.
struct TcSched {
    int G, P;
    long long U, u0, u1;
    int tile_a, a_g0, a_g1, tile_z, z_g1, n_segs;
    __host__ __device__ TcSched(int n_tiles, int G_, int P_, int b) : G(G_), P(P_) {
        U = (long long)n_tiles * G;
        u0 = b * U / P;
        u1 = (b + 1) * U / P;
        tile_a = (int)(u0 / G);
        a_g0 = (int)(u0 - (long long)tile_a * G);
        const long long len = u1 - u0;
        a_g1 = (int)((long long)a_g0 + len < G ? a_g0 + len : G);
        if (len <= 0) {
            n_segs = 0;
            tile_z = tile_a;
            z_g1 = 0;
        } else if (a_g1 - a_g0 == len) {
            n_segs = 1;
            tile_z = tile_a;
            z_g1 = a_g1;
        } else {
            tile_z = (int)((u1 - 1) / G);
            z_g1 = (int)(u1 - (long long)tile_z * G);
            n_segs = 2 + (tile_z - tile_a - 1);
        }
    }
    __host__ __device__ void seg(int i, int& tile, int& g0, int& g1) const {
        if (i == 0) {
            tile = tile_a;
            g0 = a_g0;
            g1 = a_g1;
        } else if (i == 1) {
            tile = tile_z;
            g0 = 0;
            g1 = z_g1;
        } else {
            tile = tile_a + i - 1;
            g0 = 0;
            g1 = G;
        }
    }
    // CTA that owns unit u
    __host__ __device__ int owner(long long u) const { return (int)(((u + 1) * P + U - 1) / U) - 1; }
    // workspace slot of CTA c's piece of tile t: 2 c (+ 1 when the piece does not start the CTA's range)
    __host__ __device__ int slot(int c, int t) const {
        const long long cu0 = c * U / P, t0 = (long long)t * G;
        return 2 * c + ((cu0 >= t0) ? 0 : 1);
    }
};

// dequantised fp16 pair (q - z) * s of two 4-bit codes picked from `w` by the PRMT selector
__device__ __forceinline__ uint32_t tc_dq2(uint32_t w, uint32_t magic, uint32_t sel, __half2 cz, __half2 s2) {
    uint32_t a = __byte_perm(w, magic, sel);
    __half2 v = __hmul2(__hsub2(*reinterpret_cast<__half2*>(&a), cz), s2);
    return *reinterpret_cast<uint32_t*>(&v);
}

template <int NTOK>
__global__ void __launch_bounds__(TsCfg<NTOK>::kThreads, 1) k_w4a16_ts(const __grid_constant__ W4TcParams p) {
    using C = TsCfg<NTOK>;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::kBarOff);
    uint64_t* empty = full + C::ST;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int G = p.K / kW4GroupK, n_tiles = p.N / kTcRows;
    const TcSched sch(n_tiles, G, (int)gridDim.x, (int)blockIdx.x);

    if (threadIdx.x == 0) {
        for (int i = 0; i < C::ST; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 8);             // one arrival per consumer warp
        }
        mbar_fence_init();
    }
    pdl_trigger();
    __syncthreads();

    if (warp == C::kWarpProducer) {
        // weights are constants and may be requested before the predecessor kernel has finished (PDL); x may not
        if (lane == 0) {
            const uint64_t pol = l2_evict_first_policy();
            int st = 0;
            uint32_t ph = 0;
            bool waited = false;
            for (int si = 0; si < sch.n_segs; ++si) {
                int tile, g0, g1;
                sch.seg(si, tile, g0, g1);
                for (int gi = g0; gi < g1; ++gi) {
                    mbar_wait_wd(&empty[st], ph ^ 1u, p.err, 0x100 + st);
                    mbar_expect_tx(&full[st], (uint32_t)(C::kNibGroup + 4 * 80 + C::kXGroup));
                    tma_load_4d_hint(smem + C::kNibOff + st * C::kNibGroup, &p.wmap, 0, 0, gi, tile * 4, &full[st], pol);
                    tma_load_3d_hint(smem + C::kTrOff + st * C::kTrGroup, &p.tmap, 0, gi, tile * 4, &full[st], pol);
                    if (!waited) {
                        pdl_wait();
                        waited = true;
                    }
                    uint8_t* dst = smem + C::kXOff + st * C::kXGroup;
                    tma_load_2d(dst, &p.xmap, gi * kW4GroupK, 0, &full[st]);
                    tma_load_2d(dst + NTOK * 128, &p.xmap, gi * kW4GroupK + 64, 0, &full[st]);
                    if (++st == C::ST) {
                        st = 0;
                        ph ^= 1u;
                    }
                }
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    // warp w of warpgroup wr covers rows 64 wr + 16 (w % 4) .. + 15 of the tile = ZLW4I block b = 2 wr + (w % 4) / 2 of the
    // tile, 16-row tile tt = w % 2 of that block; the thread holds rows g and g + 8 for k 2 tig, 2 tig + 1 (+ 8)
    const int b = warp >> 1, tt = warp & 1, g = lane >> 2, tig = lane & 3;
    const int m_lo = b * 32 + tt * 16 + g;                         // row in the tile; its partner is m_lo + 8
    const uint32_t sw = (uint32_t)(g >> 1) & 3u;                   // the map's 64-byte swizzle: chunk ^= (row >> 1) & 3
    const uint32_t sel = (tig & 1) ? 0x4342u : 0x4140u;            // bytes 2 tig % 4 and + 1 of a word
    const int wsel = tig >> 1;                                     // word of k 2 tig (word wsel + 2: k 2 tig + 8)
    pdl_wait();
    int st = 0;
    uint32_t ph = 0;
    for (int si = 0; si < sch.n_segs; ++si) {
        int tile, g0, g1;
        sch.seg(si, tile, g0, g1);
        float acc[NTOK / 2];
        for (int gi = g0; gi < g1; ++gi) {
            mbar_wait_wd(&full[st], ph, p.err, 0x400 + st);
            const uint8_t* nib = smem + C::kNibOff + st * C::kNibGroup + b * 2048;
            const uint8_t* tr = smem + C::kTrOff + st * C::kTrGroup + b * 80;
            const __half2 sc2 = *reinterpret_cast<const __half2*>(tr + (tt * 8 + g) * 4);
            const int zz = tr[64 + tt * 8 + g];
            const __half2 cz_lo = __float2half2_rn((float)(1024 + (zz & 0xF))), cz_hi = __float2half2_rn((float)(64 + (zz >> 4)));
            const __half2 s_lo = __half2half2(__low2half(sc2)), s_hi = __half2half2(__high2half(sc2));
            uint32_t a[8][4];
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                // 16-k step s = 2 t + hh of the group: record row (2 tt + hh) * 8 + g, 16-byte chunk t
                const int t = s >> 1, hh = s & 1;
                const uint4 wv = *reinterpret_cast<const uint4*>(nib + ((tt * 2 + hh) * 8 + g) * 64 + (((uint32_t)t ^ sw) << 4));
                const uint32_t w0 = wsel ? wv.y : wv.x, w1 = wsel ? wv.w : wv.z;
                a[s][0] = tc_dq2(w0 & 0x0f0f0f0fu, 0x64646464u, sel, cz_lo, s_lo);   // row g,     k 2 tig, 2 tig + 1
                a[s][1] = tc_dq2(w0 & 0xf0f0f0f0u, 0x54545454u, sel, cz_hi, s_hi);   // row g + 8
                a[s][2] = tc_dq2(w1 & 0x0f0f0f0fu, 0x64646464u, sel, cz_lo, s_lo);   // row g,     k 2 tig + 8, + 9
                a[s][3] = tc_dq2(w1 & 0xf0f0f0f0u, 0x54545454u, sel, cz_hi, s_hi);   // row g + 8
            }
            const uint64_t xd0 = wg_desc_sw128(smem_u32(smem + C::kXOff + st * C::kXGroup));
            wg_fence();
#pragma unroll
            for (int s = 0; s < 8; ++s)   // x: 64-k atom s / 4, 32 bytes per 16-k step
                wg_f16_rs<NTOK>(acc, a[s], xd0 + (uint64_t)((s >> 2) * ((NTOK * 128) >> 4) + (s & 3) * 2),
                                (gi > g0 || s > 0) ? 1u : 0u);
            wg_commit();
            wg_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
            if (++st == C::ST) {
                st = 0;
                ph ^= 1u;
            }
        }
        if (g0 == 0 && g1 == G) {
#pragma unroll
            for (int j = 0; j < NTOK / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    tc_epilogue_pair(p, tile * 4 + b, tt, g, 8 * j + 2 * tig + e, acc[4 * j + e], acc[4 * j + 2 + e]);
        } else {
            // a piece of a shared tile: tagged words, valid on arrival (no fence, no counter)
            uint2* wsp = p.ws + (size_t)sch.slot((int)blockIdx.x, tile) * p.M * kTcRows;
#pragma unroll
            for (int j = 0; j < NTOK / 8; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int tok = 8 * j + 2 * tig + (e & 1);
                    if (tok < p.M) tc_st_tag(wsp + (size_t)tok * kTcRows + m_lo + (e >> 1) * 8, __float_as_uint(acc[4 * j + e]), 1u);
                }
        }
    }
    // ---- shared tiles: the owners of a tile's pieces split its 16-token chunks among themselves (chunk c goes to piece
    // c mod nparts); each adds the pieces of its chunks in k order (deterministic), polling the tagged words, zeroes them for
    // the next launch and runs the epilogue.  A CTA gets here only after it has written ALL its own pieces, so nobody ever
    // waits for somebody who waits. ----
    const int ct = threadIdx.x;                                  // 0 .. 255: (token of the chunk, row pair) items
    for (int si = 0; si < sch.n_segs && si < 2; ++si) {
        int tile, g0, g1;
        sch.seg(si, tile, g0, g1);
        if (g0 == 0 && g1 == G) continue;
        const int c_first = sch.owner((long long)tile * G), c_last = sch.owner((long long)(tile + 1) * G - 1);
        const int nparts = c_last - c_first + 1, part = (int)blockIdx.x - c_first;
#pragma unroll 1
        for (int c0 = part * 16; c0 < p.M; c0 += nparts * 16) {
#pragma unroll 1
            for (int idx = ct; idx < 16 * 64; idx += 256) {
                const int tok = c0 + (idx >> 6), pr = idx & 63;
                if (tok >= p.M) continue;
                const int rb = pr >> 4, rtt = (pr >> 3) & 1, rg = pr & 7;
                const int m = rb * 32 + rtt * 16 + rg;
                float v[2] = {0.f, 0.f};
#pragma unroll 1
                for (int pp = 0; pp < nparts; ++pp) {
                    uint2* src = p.ws + ((size_t)sch.slot(c_first + pp, tile) * p.M + tok) * kTcRows + m;
                    uint2 t[2] = {tc_ld_tag(src), tc_ld_tag(src + 8)};
                    if (t[0].y != 1u || t[1].y != 1u) {   // not there yet: poll (bounded: a lost piece must not hang the GPU)
                        const long long t_start = clock64();
                        while (t[0].y != 1u || t[1].y != 1u) {
                            if (t[0].y != 1u) t[0] = tc_ld_tag(src);
                            if (t[1].y != 1u) t[1] = tc_ld_tag(src + 8);
                            if (clock64() - t_start > 4000000000ll) {
                                if (p.err) atomicExch(p.err, 0x900u + (unsigned)pp);
                                __threadfence_system();
                                __trap();
                            }
                        }
                    }
                    v[0] += __uint_as_float(t[0].x);
                    v[1] += __uint_as_float(t[1].x);
                    tc_st_tag(src, 0u, 0u);              // consumed: back to "empty"
                    tc_st_tag(src + 8, 0u, 0u);
                }
                tc_epilogue_pair(p, tile * 4 + rb, rtt, rg, tok, v[0], v[1]);
            }
        }
    }
}

// ---- host side --------------------------------------------------------------------------------------------------------
static TcDeviceState g_tc_state[64];

TcDeviceState* tc_state() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < 64) ? &g_tc_state[dev] : nullptr;
}

// allocates the per-device partial-tile workspace and sets the opt-in shared-memory sizes; must run outside stream capture
cudaError_t prepare_w4_tc() {
    TcDeviceState* st = tc_state();
    if (!st) return cudaErrorInvalidDevice;
    cudaError_t e;
    if (!st->ws) {
        if ((e = cudaMalloc((void**)&st->ws, kTcWsBytes)) != cudaSuccess) return e;
        if ((e = cudaMalloc((void**)&st->counters, (kTcMaxTiles + 16) * sizeof(unsigned))) != cudaSuccess) return e;
        if ((e = cudaMemset(st->counters, 0, (kTcMaxTiles + 16) * sizeof(unsigned))) != cudaSuccess) return e;
        st->err = st->counters + kTcMaxTiles;
        st->ws_bytes = kTcWsBytes;
        if ((e = cudaMalloc((void**)&st->ws_ll, kTcWsLlBytes)) != cudaSuccess) return e;
        if ((e = cudaMemset(st->ws_ll, 0, kTcWsLlBytes)) != cudaSuccess) return e;
        st->ws_ll_bytes = kTcWsLlBytes;
    }
#define ZL_TS_SET(NT)                                                                                             \
    if ((e = cudaFuncSetAttribute(k_w4a16_ts<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize,                     \
                                  TsCfg<NT>::kBytes)) != cudaSuccess)                                              \
        return e;
    ZL_TS_SET(32) ZL_TS_SET(64) ZL_TS_SET(128) ZL_TS_SET(256)
#undef ZL_TS_SET
    return cudaSuccess;
}

bool w4_tc_supports(int mc, int N, int K) {
    return mc >= 1 && mc <= 256 && N % kTcRows == 0 && K % kW4GroupK == 0 && N / kTcRows <= kTcMaxTiles;
}

// last watchdog code published by a tensor-core kernel on this device (0 = none); debugging aid
extern "C" unsigned zl_w4_tc_watchdog(void) {
    TcDeviceState* st = tc_state();
    unsigned v = 0;
    if (st && st->err) cudaMemcpy(&v, st->err, 4, cudaMemcpyDeviceToHost);
    return v;
}

// host view of the stream-k schedule of the wgmma kernel (the same TcSched the kernel uses), for tests: the pieces of CTA
// `cta` out of `ctas` for n_tiles x G units.  out[5 * i + 0..4] = tile, g0, g1, number of pieces of that tile, workspace slot
// of this piece (-1 for a whole tile); returns the number of pieces (<= max_pieces) or a negative error code.
extern "C" int zl_w4_tc_schedule(int n_tiles, int G, int ctas, int cta, int* out, int max_pieces) {
    if (n_tiles <= 0 || G <= 0 || ctas <= 0 || cta < 0 || cta >= ctas || !out || (long long)n_tiles * G < ctas) return ZL_ERR_INVALID_ARG;
    const TcSched sch(n_tiles, G, ctas, cta);
    if (sch.n_segs > max_pieces) return ZL_ERR_INVALID_ARG;
    for (int i = 0; i < sch.n_segs; ++i) {
        int tile, g0, g1;
        sch.seg(i, tile, g0, g1);
        const bool whole = g0 == 0 && g1 == G;
        out[5 * i + 0] = tile;
        out[5 * i + 1] = g0;
        out[5 * i + 2] = g1;
        out[5 * i + 3] = sch.owner((long long)(tile + 1) * G - 1) - sch.owner((long long)tile * G) + 1;
        out[5 * i + 4] = whole ? -1 : sch.slot(cta, tile);
    }
    return sch.n_segs;
}

// grid override: ZL_TC_CTAS in the environment, or zl_w4_tc_set_splits(n) = "at least n pieces per tile" (tests exercise
// the partial-tile exchange on small shapes); 0 = automatic
static int g_tc_splits = -2;
static int tc_force_splits() {
    if (g_tc_splits == -2) {
        const char* e = getenv("ZL_TC_SPLITS");
        g_tc_splits = e ? atoi(e) : 0;
    }
    return g_tc_splits;
}
extern "C" int zl_w4_tc_set_splits(int splits) {
    g_tc_splits = splits < 0 ? 0 : splits;
    return ZL_OK;
}

// number of CTAs: every SM when each gets at least kMinUnits (tile, group) units, fewer for small GEMMs (every extra piece
// of a tile is an fp32 round trip through L2 for its last arriver)
static int tc_pick_ctas(int n_tiles, int G) {
    static const int env_ctas = getenv("ZL_TC_CTAS") ? atoi(getenv("ZL_TC_CTAS")) : 0;
    static const int min_units = getenv("ZL_TC_MIN_UNITS") ? atoi(getenv("ZL_TC_MIN_UNITS")) : 8;
    const int sms = device_sm_count();
    const long long U = (long long)n_tiles * G;
    long long P = sms;
    const int forced = tc_force_splits();
    if (env_ctas > 0) {
        P = env_ctas;
    } else if (forced > 0) {
        P = (long long)n_tiles * forced;
    } else if (U / P < min_units) {
        P = U / min_units;
        if (P < n_tiles) P = n_tiles;
    }
    if (P > sms) P = sms;
    if (P > U) P = U;
    if (P < 1) P = 1;
    return (int)P;
}

cudaError_t launch_w4_tc(const W4Params& p, bool pdl, cudaStream_t stream) {
    TcDeviceState* st = tc_state();
    if (!st || !st->ws) return cudaErrorNotSupported;
    const int ntok = p.mc <= 32 ? 32 : p.mc <= 64 ? 64 : p.mc <= 128 ? 128 : 256;
    const int n_tiles = p.N / kTcRows, G = p.K / kW4GroupK;
    W4TcParams q;
    if (!tc_make_map_2d(&q.xmap, p.x, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (uint64_t)p.mc, (uint64_t)p.K, (uint64_t)p.ldx * 2,
                        (uint32_t)ntok))
        return cudaErrorInvalidValue;
    {
        // the weight maps depend only on (address, N, K): encode once per weight matrix (cuTensorMapEncodeTiled costs
        // microseconds of host time per call)
        struct WMaps {
            CUtensorMap w, t;
        };
        static std::map<std::tuple<const void*, int, int>, WMaps> cache;
        static std::mutex mu;
        std::lock_guard<std::mutex> lock(mu);
        const auto key = std::make_tuple((const void*)p.packed, p.N, p.K);
        auto it = cache.find(key);
        if (it == cache.end()) {
            const uint64_t nb = (uint64_t)p.N / 32;
            const uint64_t wd[4] = {16, 32, (uint64_t)G, nb}, wstr[3] = {64, (uint64_t)kW4BlockBytes, (uint64_t)G * kW4BlockBytes};
            const uint32_t wbox[4] = {16, 32, 1, 4};
            const uint64_t td[3] = {20, (uint64_t)G, nb}, tstr[2] = {(uint64_t)kW4BlockBytes, (uint64_t)G * kW4BlockBytes};
            const uint32_t tbox[3] = {20, 1, 4};
            WMaps m;
            if (!tc_make_map_nd(&m.w, p.packed, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4, wd, wstr, wbox, CU_TENSOR_MAP_SWIZZLE_64B) ||
                !tc_make_map_nd(&m.t, p.packed + kW4ScaleOff, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, td, tstr, tbox,
                                CU_TENSOR_MAP_SWIZZLE_NONE))
                return cudaErrorInvalidValue;
            if (cache.size() > 4096) cache.clear();
            it = cache.emplace(key, m).first;
        }
        q.wmap = it->second.w;
        q.tmap = it->second.t;
    }
    q.packed = p.packed;
    q.bias = p.bias;
    q.residual = p.residual;
    q.y = p.y;
    q.M = p.mc;
    q.N = p.N;
    q.K = p.K;
    q.epi = p.epi;
    q.ws = st->ws_ll;
    q.err = st->err;
    q.cos = p.cos;
    q.sin = p.sin;
    q.q_out = p.q_out;
    q.token_batch = p.token_batch;
    q.placement = p.placement;
    q.k_addrs = p.k_addrs;
    q.v_addrs = p.v_addrs;
    q.num_heads = p.num_heads;
    q.num_kv_heads = p.num_kv_heads;
    q.dim_head = p.dim_head;
    const int ctas = tc_pick_ctas(n_tiles, G);
    if ((size_t)2 * ctas * p.mc * kTcRows * 8 > st->ws_ll_bytes) return cudaErrorInvalidValue;
    const dim3 grid(ctas);
    switch (ntok) {
        case 32: return launch(k_w4a16_ts<32>, grid, dim3(TsCfg<32>::kThreads), (size_t)TsCfg<32>::kBytes, stream, pdl, q);
        case 64: return launch(k_w4a16_ts<64>, grid, dim3(TsCfg<64>::kThreads), (size_t)TsCfg<64>::kBytes, stream, pdl, q);
        case 128: return launch(k_w4a16_ts<128>, grid, dim3(TsCfg<128>::kThreads), (size_t)TsCfg<128>::kBytes, stream, pdl, q);
        default: return launch(k_w4a16_ts<256>, grid, dim3(TsCfg<256>::kThreads), (size_t)TsCfg<256>::kBytes, stream, pdl, q);
    }
}

}  // namespace zl
