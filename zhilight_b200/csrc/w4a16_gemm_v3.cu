// W4A16 skinny GEMM, exact-integer variant (ZLW4I layout): the default for small M.
//
// Why: a decode GEMM must consume ~14 weight bytes per cycle per SM to keep up with an H100's HBM3.  The classic
// "dequantise int4 -> fp16 on the CUDA cores, then HMMA" recipe (our v1/v2 kernels, Marlin, the reference's
// GEMV) costs ~10 issue slots per packed word, which makes the kernel ISSUE-bound before it is HBM-bound
// (measured on the previous target).  Here the int4 weights never
// become floating point:
//   * activations are decomposed once per CTA into a block-floating-point integer  x_k = 2^e_g * m_k,
//     m_k a 16-bit integer per 128-group (error <= 2^-16 of the group maximum, far below fp16's own 2^-11),
//     split into a signed high byte and an unsigned low byte;
//   * a packed weight word turns into two IMMA A registers with two LOP3s (w & 0x0f0f0f0f, w & 0xf0f0f0f0 --
//     the odd nibbles stay multiplied by 16 and the factor is folded into that row's scale);
//   * sum_k q_k * m_k is accumulated EXACTLY in int32 by mma.sync.m16n8k32 (u8 x s8 and u8 x u8), the zero
//     point is removed with the exact group sum of m, and only then one fp32 multiply by
//     scale[row,g] * 2^e_g happens per group.
// ~3 issue slots per word instead of ~10, and the result is closer to the exact product than either the fp16
// reference kernel or our fp16 path.  Same ring / persistence / fused prologue+epilogues as v2.
#include "common.cuh"
#include "w4_layout.cuh"
#include "w4_params.h"
#include "comm_dev.cuh"

#include <cstdlib>

namespace zl {

__device__ __forceinline__ void imma_u8s8(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void imma_u8u8(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Shared-memory plan.  A CTA holds SUBS independent "sub-CTAs" of WARPS warps; each sub-CTA walks its own stream
// of 32-row tiles (k split over its WARPS warps, private bulk-TMA rings, own named barrier for the split-k
// reduction), while the integer decomposition of the activations is staged ONCE per CTA by all warps together:
//   wide : SUBS=2 x 8 warps, 5-stage rings  (N/32 > #SMs: qkv, gate/up)  -- two tile pipelines per SM
//   tall : SUBS=1 x 16 warps, 4-stage rings (N/32 <= #SMs: o_proj, down) -- k split 16 ways
// RT = token rows kept in the split-k reduction buffers (even, >= mc): small batches shrink them to make room for
// deeper rings -- the tile loop is latency-bound on ring depth (4 -> 5 stages is worth ~25 %).
template <int NT, int WARPS, int SUBS, int STAGES, int RT = NT * 8>
struct V3Smem {
    static constexpr int kWarpsTotal = WARPS * SUBS;
    static constexpr int kRingBytes = kWarpsTotal * STAGES * kW4BlockBytes;
    static constexpr int kRedBufs = (NT == 1) ? 2 : 1;
    static constexpr int kRedFloats = WARPS * RT * 32;                     // per sub-CTA, per buffer
    static constexpr int kBarOff = kRingBytes;
    static constexpr int kRedOff = kBarOff + kWarpsTotal * STAGES * 8;
    static constexpr int kSsOff = kRedOff + SUBS * kRedBufs * kRedFloats * 4;   // [warps total][NT*8] sum x^2 | [warps total][NT*8] poison
    static constexpr int kRstdOff = kSsOff + 2 * kWarpsTotal * NT * 8 * 4;      // [NT*8] rstd | [NT*8] poison
    static constexpr int kXOff = (kRstdOff + 2 * NT * 8 * 4 + 127) & ~127;
    static constexpr int kBytes = kXOff;
};
// staged activations (whole K): mc rows of hi bytes, mc rows of lo bytes, then the group table
__host__ __device__ inline int v3_row_bytes(int K) { return K + 16; }   // +16: conflict-free LDS.128 across tokens
__host__ __device__ inline int v3_stage_bytes(int mc, int K) {
    return 2 * mc * v3_row_bytes(K) + (K / kW4GroupK) * mc * 8;
}

__device__ __forceinline__ void sub_barrier(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// PACK block math for NB blocks of one warp at once (NB = 2: two independent dependency chains interleave).
template <int NB>
__device__ __forceinline__ void pack_blocks(const W4Params& p, const uint8_t* ring, uint64_t* bars, const uint8_t* xs_hi,
                                            const uint8_t* xs_lo, const int2* xs_tab, int row_b, const int* slot,
                                            const uint32_t* parity, const int* gi, int g, int t, int lane,
                                            float (&acc)[2][1][4]) {
    // B fragment column n = g carries token g>>1, digit g&1 (0: high, 1: low); 32 contiguous bytes per lane
    uint4 bv[NB][2];
    int2 tb[NB];
    const int tok = g >> 1;
#pragma unroll
    for (int u = 0; u < NB; ++u) {
        if (tok < p.mc) {
            const uint8_t* pp = ((g & 1) ? xs_lo : xs_hi) + tok * row_b + gi[u] * 128 + t * 32;
            bv[u][0] = *reinterpret_cast<const uint4*>(pp);
            bv[u][1] = *reinterpret_cast<const uint4*>(pp + 16);
        } else {
            bv[u][0] = bv[u][1] = make_uint4(0, 0, 0, 0);
        }
        // C columns (2t, 2t+1) = (high, low) digit sums of token t: this lane finishes token t
        tb[u] = t < p.mc ? xs_tab[gi[u] * p.mc + t] : make_int2(0, 0);
    }
    const uint8_t* blk[NB];
#pragma unroll
    for (int u = 0; u < NB; ++u) {
        mbar_wait(&bars[slot[u]], parity[u]);
        blk[u] = ring + slot[u] * kW4BlockBytes;
    }
    int cc[NB][2][4];
#pragma unroll
    for (int u = 0; u < NB; ++u)
#pragma unroll
        for (int tt = 0; tt < 2; ++tt)
#pragma unroll
            for (int c = 0; c < 4; ++c) cc[u][tt][c] = 0;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        uint4 wv[NB][2];
#pragma unroll
        for (int u = 0; u < NB; ++u)
#pragma unroll
            for (int tt = 0; tt < 2; ++tt)
                wv[u][tt] = *reinterpret_cast<const uint4*>(blk[u] + ((tt * 2 + hh) * 32 + lane) * 16);
#pragma unroll
        for (int jp = 0; jp < 2; ++jp) {
            const int j = hh * 2 + jp;   // k-step 0..3
#pragma unroll
            for (int tt = 0; tt < 2; ++tt) {
#pragma unroll
                for (int u = 0; u < NB; ++u) {
                    const uint32_t w0 = jp ? wv[u][tt].z : wv[u][tt].x;
                    const uint32_t w1 = jp ? wv[u][tt].w : wv[u][tt].y;
                    const uint32_t a[4] = {w0 & 0x0f0f0f0fu, w0 & 0xf0f0f0f0u, w1 & 0x0f0f0f0fu, w1 & 0xf0f0f0f0u};
                    const uint4 v = bv[u][j >> 1];
                    imma_u8s8(cc[u][tt], a, (j & 1) ? v.z : v.x, (j & 1) ? v.w : v.y);
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < NB; ++u) {   // blocks in k order: the fp32 accumulation order does not depend on NB
        const float sgf = __int_as_float(tb[u].y);
#pragma unroll
        for (int tt = 0; tt < 2; ++tt) {
            const __half2 sc = *reinterpret_cast<const __half2*>(blk[u] + kW4ScaleOff + (tt * 8 + g) * 4);
            const int zz = blk[u][kW4ZeroOff + tt * 8 + g];
            const int z_lo = zz & 0xF, z_hi16 = zz & 0xF0;          // zero of row g ; 16 * zero of row g+8
            const float s_lo = __low2float(sc), s_hi = __high2float(sc) * 0.0625f;
            const int r0 = cc[u][tt][0] * 256 + cc[u][tt][1] - z_lo * tb[u].x;      // row g
            const int r1 = cc[u][tt][2] * 256 + cc[u][tt][3] - z_hi16 * tb[u].x;    // row g + 8 (x16 folded in s_hi)
            acc[tt][0][0] = fmaf((float)r0, s_lo * sgf, acc[tt][0][0]);
            acc[tt][0][2] = fmaf((float)r1, s_hi * sgf, acc[tt][0][2]);
        }
    }
}

// PACK (mc <= 4): the MMA N dimension (8 columns) is mostly padding at tiny batch, so the two 8-bit digits of the
// 16-bit activation mantissas share ONE IMMA: column 2i carries token i's high digit, column 2i+1 its low digit, both
// signed (m = 256*hi' + lo', lo' = int8(m & 0xff), hi' = (m + 128) >> 8, |m| <= 2^14).  Half the IMMAs, half the B
// loads, and the per-group int->float epilogue only touches real tokens.
template <int NT, bool NORM, int WARPS, int SUBS, int STAGES, int RT = NT * 8, bool PACK = false, int TPX = 0>
__global__ void __launch_bounds__(WARPS * SUBS * 32, 1) k_w4a16_v3(const W4Params p) {
    using S = V3Smem<NT, WARPS, SUBS, STAGES, RT>;
    // the tensor-parallel exchange code is compiled only into the TPX instantiations: carried as a run-time branch it cost
    // every launch 10-20 registers (to the 128-register cap of the 512-thread CTA) and ~5 % of a single-GPU decode step
    constexpr int tp_mode = TPX;   // 0 none, 1 reduce-in while staging, 2 push from the epilogue (== p.tp_mode, checked by the launcher)
    constexpr int WT = WARPS * SUBS;
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sub = warp / WARPS, wl = warp % WARPS;   // sub-CTA, warp within it
    const int stid = threadIdx.x - sub * (WARPS * 32);  // thread index within the sub-CTA
    const int g = lane >> 2, t = lane & 3;
    const int G = p.K / kW4GroupK;
    const int g_begin = (wl * G) / WARPS;
    const int g_end = ((wl + 1) * G) / WARPS;
    const int ng = g_end - g_begin;
    const int n_tiles = p.N / 32;
    const int tile0 = (int)blockIdx.x * SUBS + sub;
    const int tile_stride = (int)gridDim.x * SUBS;
    const int my_tiles = tile0 < n_tiles ? (n_tiles - tile0 + tile_stride - 1) / tile_stride : 0;
    const int total = my_tiles * ng;

    uint8_t* ring = smem + warp * (STAGES * kW4BlockBytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kBarOff) + warp * STAGES;
    float* red = reinterpret_cast<float*>(smem + S::kRedOff) + sub * (S::kRedBufs * S::kRedFloats);
    float* s_ss = reinterpret_cast<float*>(smem + S::kSsOff);
    float* s_rstd = reinterpret_cast<float*>(smem + S::kRstdOff);
    // Inf / NaN activations: the integer decomposition cannot carry them, so a group whose maximum is non-finite
    // poisons every output of its token with NaN (the reference GEMV, q_gemm_k_major.cu:127-173, yields NaN or +-Inf
    // there) instead of silently contributing zero.
    float* s_pw = s_ss + WT * (NT * 8);       // per (warp, token): 0 or NaN
    float* s_poison = s_rstd + NT * 8;        // per token
    const int row_b = v3_row_bytes(p.K);
    uint8_t* xs_hi = smem + S::kXOff;                                    // [tok][row_b]
    uint8_t* xs_lo = xs_hi + p.mc * row_b;                               // [tok][row_b]
    int2* xs_tab = reinterpret_cast<int2*>(xs_lo + p.mc * row_b);        // [group][tok] {sum m, bits of 2^e}

    // producer cursor (lane 0): next ring item = (tile p_tile, group p_g) -> slot p_slot
    int p_issued = 0, p_tile = tile0, p_g = 0, p_slot = 0;
    const uint64_t pol = l2_evict_first_policy();
    auto issue_next = [&]() {
        mbar_expect_tx(&bars[p_slot], kW4BlockBytes);
        bulk_g2s_hint(ring + p_slot * kW4BlockBytes, p.packed + ((size_t)p_tile * G + g_begin + p_g) * kW4BlockBytes,
                      kW4BlockBytes, &bars[p_slot], pol);
        ++p_issued;
        if (++p_slot == STAGES) p_slot = 0;
        if (++p_g == ng) {
            p_g = 0;
            p_tile += tile_stride;
        }
    };

    // debug timeline: dbg & 2 -> one record per LAUNCH (CTA 0 claims a slot: trace[0] is the launch counter),
    // otherwise one record per CTA
    unsigned long long* tr = nullptr;
    if (p.trace) {
        if (p.dbg & 2) {
            if (blockIdx.x == 0 && threadIdx.x == 0)
                tr = p.trace + 8 + (size_t)atomicAdd(p.trace, 1ull) * 16;
        } else {
            tr = p.trace + (size_t)blockIdx.x * 16;
        }
    }
    int tr_n = 0;
    auto stamp = [&]() {
        if (tr && threadIdx.x == 0 && tr_n < 16) tr[tr_n++] = globaltimer_ns();
    };
    stamp();
    pdl_trigger();
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) mbar_init(&bars[s], 1);
        mbar_fence_init();
#pragma unroll
        for (int s = 0; s < STAGES; ++s)
            if (s < total) issue_next();
        // software-managed L2: start pulling the weights of a LATER kernel of the chain into the 126 MB L2 now, so
        // that HBM keeps streaming while this kernel and its neighbours sit in their latency-bound phases
        if (p.pf_ptr && !(p.dbg & 4))
            l2_prefetch_share(p.pf_ptr, (size_t)p.pf_bytes, (int)blockIdx.x * WT + warp, (int)gridDim.x * WT);
    }
    if (p.pf_ptr && (p.dbg & 4))
        l2_prefetch_lines(p.pf_ptr, (size_t)p.pf_bytes, (int)blockIdx.x * WT + warp, (int)gridDim.x * WT, lane);
    // staging assignment: group gi -> warp gi % WT.  RMSNorm weights are constants: fetch them before the wait.
    constexpr int kMaxNg = 8;   // groups per warp kept in registers during staging (K <= 8*WT*128)
    uint2 lnw[kMaxNg];
    if (NORM) {
#pragma unroll
        for (int gl = 0; gl < kMaxNg; ++gl) {
            const int gi = warp + gl * WT;
            if (gi < G)
                lnw[gl] = (p.dbg & 16) ? make_uint2(0x3c003c00u, 0x3c003c00u)   // timing probe: 1.0h (results are wrong)
                                       : *reinterpret_cast<const uint2*>(p.ln_w + gi * kW4GroupK + lane * 4);
        }
    }
    __syncwarp();
    stamp();
    pdl_wait();   // everything above touched only constants; x / residual / KV come from predecessor kernels
    stamp();

    // ---- tensor-parallel reduce-in: the partial sums of the previous row-parallel GEMM arrive in this rank's inbox as
    // 8-byte words {2 x fp16, tag}; a word is valid once its tag is the tag of this exchange (comm_dev.cuh) -- no flags,
    // no fences: the staging loop below polls the words it needs ----
    const CommDev* tp = static_cast<const CommDev*>(p.tp_cd);
    const uint8_t* tp_slots = nullptr;   // [ws][2 * slot_bytes] of the exchange's parity
    size_t tp_slot_bytes = 0;            // bytes of one source's tagged slot
    int tp_ws = 0;
    uint32_t tp_tag = 0;
    int tp_parity = 0;
    if (tp_mode != 0) {
        tp_ws = tp->ws;
        tp_slot_bytes = 2 * tp->slot_bytes;
        const unsigned int step = *reinterpret_cast<volatile unsigned int*>(tp->ll_step);
        const int idx = p.tp_index & 511;
        tp_tag = comm_ll_tag(step, idx);
        // consecutive exchanges alternate between the two slots, across step boundaries too: bit 9 of tp_index says that the
        // step has an odd number of exchanges (then the parity sequence flips every step; tests/test_dist_cpu.py models why)
        tp_parity = (idx + ((p.tp_index >> 9) & 1) * (int)(step & 1u)) & 1;
    }
    if (tp_mode == 1)
        tp_slots = tp->inbox[tp->rank] + comm_ll_offset(tp_ws, tp->slot_bytes) + (size_t)tp_parity * tp_ws * tp_slot_bytes;

    // ---- stage the activations as block-floating-point integers, once per CTA ----
    for (int tok = 0; tok < p.mc; ++tok) {
        uint2 raw[kMaxNg];
#pragma unroll
        for (int gl = 0; gl < kMaxNg; ++gl) {
            const int gi = warp + gl * WT;
            if (gi < G) raw[gl] = ld_cg_u2(p.x + (size_t)tok * p.ldx + gi * kW4GroupK + lane * 4);
        }
        if (tp_mode == 1) {
            // x := T(T(sum_r partial_r) + x): fp32 sum in rank order (identical on every rank and CTA), the reference's
            // reduce_sum + element_add_scale rounding points (model_context.cpp:203-243, block_kernel.cu:7-17).  One group
            // at a time: the accumulators of all groups at once cost the 512-thread CTA its register budget.
            // element i of token tok lives in word (tok * K + i) / 2 of the source's slot; this lane needs 4 elements = 2 words
            const uint8_t* src0 = tp_slots + ((size_t)tok * p.K + lane * 4) * 4;
#pragma unroll
            for (int gl = 0; gl < kMaxNg; ++gl) {
                const int gi = warp + gl * WT;
                if (gi < G) {
                    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
                    for (int r = 0; r < tp_ws; ++r) {
                        const uint8_t* src = src0 + (size_t)r * tp_slot_bytes + (size_t)gi * kW4GroupK * 4;
                        uint4 t = ld_ll2(src);
                        if (t.y != tp_tag || t.w != tp_tag) {   // not there yet: poll (bounded: a lost peer must not hang the GPU)
                            const long long t0 = clock64();
                            do {
                                t = ld_ll2(src);
                                if (clock64() - t0 > 4000000000ll) __trap();
                            } while (t.y != tp_tag || t.w != tp_tag);
                        }
                        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&t.x));
                        const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&t.z));
                        a0 += a.x;
                        a1 += a.y;
                        a2 += b.x;
                        a3 += b.y;
                    }
                    const __half2 h01 = __hadd2(__floats2half2_rn(a0, a1), *reinterpret_cast<__half2*>(&raw[gl].x));
                    const __half2 h23 = __hadd2(__floats2half2_rn(a2, a3), *reinterpret_cast<__half2*>(&raw[gl].y));
                    raw[gl].x = *reinterpret_cast<const uint32_t*>(&h01);
                    raw[gl].y = *reinterpret_cast<const uint32_t*>(&h23);
                    if (blockIdx.x == 0)
                        *reinterpret_cast<uint2*>(p.tp_h_out + (size_t)tok * p.K + gi * kW4GroupK + lane * 4) = raw[gl];
                }
            }
        }
        float sq = 0.f;
        bool bad = false;
#pragma unroll
        for (int gl = 0; gl < kMaxNg; ++gl) {
            const int gi = warp + gl * WT;
            if (gi < G) {
                __half2 h01 = *reinterpret_cast<__half2*>(&raw[gl].x), h23 = *reinterpret_cast<__half2*>(&raw[gl].y);
                if (NORM) {
                    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
                    sq = fmaf(f01.x, f01.x, sq);
                    sq = fmaf(f01.y, f01.y, sq);
                    sq = fmaf(f23.x, f23.x, sq);
                    sq = fmaf(f23.y, f23.y, sq);
                    h01 = __hmul2(h01, *reinterpret_cast<const __half2*>(&lnw[gl].x));
                    h23 = __hmul2(h23, *reinterpret_cast<const __half2*>(&lnw[gl].y));
                }
                const float2 a = __half22float2(h01), b = __half22float2(h23);
                // non-negative floats order like their bit patterns (and NaN patterns sort above Inf, which fmaxf would
                // drop): integer maxima, then one REDUX instead of a shuffle tree
                const uint32_t amax_l = max(max(__float_as_uint(fabsf(a.x)), __float_as_uint(fabsf(a.y))),
                                            max(__float_as_uint(fabsf(b.x)), __float_as_uint(fabsf(b.y))));
                const uint32_t amax_bits = __reduce_max_sync(0xffffffffu, amax_l);
                // 2^e with m = x * 2^-e in (-2^15, 2^15): e = floor(log2 amax) - 14
                const uint32_t ex = (amax_bits >> 23) & 0xffu;
                const bool zero = ex < 20u || ex == 0xffu;   // all-zero group -> 0; non-finite group -> poisons the token
                bad |= ex == 0xffu;                          // (a NaN's bit pattern is above Inf's: REDUX max keeps it)
                // PACK keeps one bit of headroom (|m| <= 2^14) so that the rounded-up high digit still fits int8
                constexpr uint32_t kE = PACK ? 13u : 14u;
                const float sg = zero ? 1.0f : __uint_as_float((ex - kE) << 23);
                const float inv = zero ? 0.0f : __uint_as_float((254u + kE - ex) << 23);
                const int m0 = __float2int_rn(a.x * inv), m1 = __float2int_rn(a.y * inv);
                const int m2 = __float2int_rn(b.x * inv), m3 = __float2int_rn(b.y * inv);
                // byte 0 of each m -> lo, byte 1 -> hi (two's complement high byte == floor(m / 256)): 6 PRMTs.
                // PACK: lo is read as SIGNED, so hi = floor((m + 128) / 256) = byte 1 of m + 128.
                constexpr int kR = PACK ? 128 : 0;
                const uint32_t lo = __byte_perm(__byte_perm((uint32_t)m0, (uint32_t)m1, 0x0040),
                                                __byte_perm((uint32_t)m2, (uint32_t)m3, 0x0040), 0x5410);
                const uint32_t hi = __byte_perm(__byte_perm((uint32_t)(m0 + kR), (uint32_t)(m1 + kR), 0x0051),
                                                __byte_perm((uint32_t)(m2 + kR), (uint32_t)(m3 + kR), 0x0051), 0x5410);
                *reinterpret_cast<uint32_t*>(xs_hi + tok * row_b + gi * 128 + lane * 4) = hi;
                *reinterpret_cast<uint32_t*>(xs_lo + tok * row_b + gi * 128 + lane * 4) = lo;
                const int sm = __reduce_add_sync(0xffffffffu, m0 + m1 + m2 + m3);
                if (lane == 0) xs_tab[gi * p.mc + tok] = make_int2(sm, (int)__float_as_uint(sg));
            }
        }
        if (NORM) {
            sq = warp_sum(sq);
            if (lane == 0) s_ss[warp * (NT * 8) + tok] = sq;
        }
        if (lane == 0) s_pw[warp * (NT * 8) + tok] = bad ? __int_as_float(0x7fc00000) : 0.f;
    }
    if (p.dbg & 8) stamp();   // warp 0 finished its groups (loads landed + quantised)
    __syncthreads();
    if (p.dbg & 8) stamp();   // all warps staged
    if (threadIdx.x < p.mc) {
        float po = 0.f;
#pragma unroll
        for (int w = 0; w < WT; ++w) po += s_pw[w * (NT * 8) + threadIdx.x];
        s_poison[threadIdx.x] = po;
        if (NORM) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < WT; ++w) v += s_ss[w * (NT * 8) + threadIdx.x];
            s_rstd[threadIdx.x] = rsqrtf(v / (float)p.K + p.eps);
        }
    }
    __syncthreads();
    stamp();

    // tensor-parallel push: tagged slot (parity of the exchange index, this rank) of every rank's inbox
    size_t tp_my_slot = 0;
    if (tp_mode == 2)
        tp_my_slot = comm_ll_offset(tp_ws, tp->slot_bytes) + ((size_t)tp_parity * tp_ws + tp->rank) * tp_slot_bytes;

    int c_slot = 0;
    uint32_t c_parity = 0;
    for (int ti = 0; ti < my_tiles; ++ti) {
        const int st = tile0 + ti * tile_stride;
        float acc[2][NT][4];
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < NT; ++b)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;

        int i = 0;
        if constexpr (PACK) {
            // two blocks in flight per warp: their smem loads, IMMA chains and epilogues interleave (the per-block
            // dependency chain, not issue slots or HBM, is what a single block per warp leaves exposed)
            for (; i + 2 <= ng; i += 2) {
                int ss[2], gg[2];
                uint32_t pp[2];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    ss[u] = c_slot;
                    pp[u] = c_parity;
                    if (++c_slot == STAGES) {
                        c_slot = 0;
                        c_parity ^= 1u;
                    }
                    gg[u] = g_begin + i + u;
                }
                pack_blocks<2>(p, ring, bars, xs_hi, xs_lo, xs_tab, row_b, ss, pp, gg, g, t, lane, acc);
                __syncwarp();
                if (lane == 0) {
                    if (p_issued < total) issue_next();
                    if (p_issued < total) issue_next();
                }
            }
        }
        for (; i < ng; ++i) {
            const int s = c_slot;
            const uint32_t parity = c_parity;
            if (++c_slot == STAGES) {
                c_slot = 0;
                c_parity ^= 1u;
            }
            const int gi = g_begin + i;
            if constexpr (PACK) {
                pack_blocks<1>(p, ring, bars, xs_hi, xs_lo, xs_tab, row_b, &s, &parity, &gi, g, t, lane, acc);
            } else {
                // B fragments: 32 contiguous bytes of each piece per lane
                uint4 bh[NT][2], bl[NT][2];
                int2 tab[NT][2];
    #pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    const int tok = nt * 8 + g;
                    if (tok < p.mc) {
                        const uint8_t* ph = xs_hi + tok * row_b + gi * 128 + t * 32;
                        const uint8_t* pl = xs_lo + tok * row_b + gi * 128 + t * 32;
                        bh[nt][0] = *reinterpret_cast<const uint4*>(ph);
                        bh[nt][1] = *reinterpret_cast<const uint4*>(ph + 16);
                        bl[nt][0] = *reinterpret_cast<const uint4*>(pl);
                        bl[nt][1] = *reinterpret_cast<const uint4*>(pl + 16);
                    } else {
                        bh[nt][0] = bh[nt][1] = bl[nt][0] = bl[nt][1] = make_uint4(0, 0, 0, 0);
                    }
                    // group table of the two tokens this lane's accumulators belong to (C columns 2t, 2t+1)
    #pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int tc = nt * 8 + 2 * t + e;
                        tab[nt][e] = tc < p.mc ? xs_tab[gi * p.mc + tc] : make_int2(0, 0);
                    }
                }

                mbar_wait(&bars[s], parity);
                const uint8_t* blk = ring + s * kW4BlockBytes;
                if (p.dbg & 1) {
                    acc[0][0][0] += __uint_as_float(*reinterpret_cast<const uint32_t*>(blk + lane * 4)) * 1e-30f;
                } else {
                    int ah[2][NT][4], al[2][NT][4];
    #pragma unroll
                    for (int tt = 0; tt < 2; ++tt)
    #pragma unroll
                        for (int nt = 0; nt < NT; ++nt)
    #pragma unroll
                            for (int c = 0; c < 4; ++c) ah[tt][nt][c] = al[tt][nt][c] = 0;
    #pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        uint4 wv[2];
    #pragma unroll
                        for (int tt = 0; tt < 2; ++tt)
                            wv[tt] = *reinterpret_cast<const uint4*>(blk + ((tt * 2 + hh) * 32 + lane) * 16);
    #pragma unroll
                        for (int jp = 0; jp < 2; ++jp) {
                            const int j = hh * 2 + jp;   // k-step 0..3
    #pragma unroll
                            for (int tt = 0; tt < 2; ++tt) {   // the two 16-row tiles interleave: independent chains
                                const uint32_t w0 = jp ? wv[tt].z : wv[tt].x;
                                const uint32_t w1 = jp ? wv[tt].w : wv[tt].y;
                                const uint32_t a[4] = {w0 & 0x0f0f0f0fu, w0 & 0xf0f0f0f0u, w1 & 0x0f0f0f0fu,
                                                       w1 & 0xf0f0f0f0u};
    #pragma unroll
                                for (int nt = 0; nt < NT; ++nt) {
                                    const uint4 vh = bh[nt][j >> 1], vl = bl[nt][j >> 1];
                                    imma_u8s8(ah[tt][nt], a, (j & 1) ? vh.z : vh.x, (j & 1) ? vh.w : vh.y);
                                    imma_u8u8(al[tt][nt], a, (j & 1) ? vl.z : vl.x, (j & 1) ? vl.w : vl.y);
                                }
                            }
                        }
                    }
                    // exact integer group result, then one fp32 multiply-add per element
    #pragma unroll
                    for (int tt = 0; tt < 2; ++tt) {
                        const __half2 sc = *reinterpret_cast<const __half2*>(blk + kW4ScaleOff + (tt * 8 + g) * 4);
                        const int zz = blk[kW4ZeroOff + tt * 8 + g];
                        const int z_lo = zz & 0xF, z_hi16 = zz & 0xF0;          // zero of row g ; 16 * zero of row g+8
                        const float s_lo = __low2float(sc), s_hi = __high2float(sc) * 0.0625f;
    #pragma unroll
                        for (int nt = 0; nt < NT; ++nt) {
    #pragma unroll
                            for (int c = 0; c < 4; ++c) {
                                const int2 tb = tab[nt][c & 1];
                                const int zc = (c >> 1) ? z_hi16 : z_lo;
                                const int r = ah[tt][nt][c] * 256 + al[tt][nt][c] - zc * tb.x;
                                const float f = ((c >> 1) ? s_hi : s_lo) * __int_as_float(tb.y);
                                acc[tt][nt][c] = fmaf((float)r, f, acc[tt][nt][c]);
                            }
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0 && p_issued < total) issue_next();   // refills the slot just drained (p_slot == s)
        }

        // ---- split-k reduction across the warps of this sub-CTA + epilogue ----
        float* rbuf = red + (S::kRedBufs == 2 ? (ti & 1) * S::kRedFloats : 0);
        float* myred = rbuf + wl * (RT * 32);
#pragma unroll
        for (int tt = 0; tt < 2; ++tt)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const int row = tt * 16 + g;
                if constexpr (PACK) {   // lane t holds token t: acc[.][0][0] = row g, acc[.][0][2] = row g + 8
                    if (t < RT) {
                        myred[t * 32 + row] = acc[tt][0][0];
                        myred[t * 32 + row + 8] = acc[tt][0][2];
                    }
                    continue;
                }
                const int tok = nt * 8 + 2 * t;
                if (RT == NT * 8 || tok < RT) {
                    myred[tok * 32 + row] = acc[tt][nt][0];
                    myred[(tok + 1) * 32 + row] = acc[tt][nt][1];
                    myred[tok * 32 + row + 8] = acc[tt][nt][2];
                    myred[(tok + 1) * 32 + row + 8] = acc[tt][nt][3];
                }
            }
        sub_barrier(1 + sub, WARPS * 32);

        auto sum_red = [&](int idx) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < WARPS; ++w) v += rbuf[w * (RT * 32) + idx];
            return v;
        };
        const int n0 = st * 32;
        constexpr int kSubThreads = WARPS * 32;
        if (p.epi == ZL_EPI_SWIGLU) {
            const int n_out = p.N / 2;
            for (int e = stid; e < p.mc * 16; e += kSubThreads) {
                const int tok = e >> 4, oc = e & 15;
                const int rg = (oc >> 3) * 16 + (oc & 7);
                float gate = sum_red(tok * 32 + rg);
                float up = sum_red(tok * 32 + rg + 8);
                if (NORM) {
                    gate *= s_rstd[tok];
                    up *= s_rstd[tok];
                }
                gate += s_poison[tok];
                up += s_poison[tok];
                if (p.bias) {
                    gate += __half2float(p.bias[n0 + rg]);
                    up += __half2float(p.bias[n0 + rg + 8]);
                }
                const float gr = __half2float(__float2half_rn(gate));
                const float ur = __half2float(__float2half_rn(up));
                p.y[(size_t)tok * n_out + st * 16 + oc] = __float2half_rn(silu_f(gr) * ur);
            }
        } else if (p.epi == ZL_EPI_QKV_ROPE) {
            const int d = p.dim_head, half_dim = d / 2;
            const int tiles_per_head = d / 32;
            const int head = st / tiles_per_head, jt = st % tiles_per_head;
            for (int e = stid; e < p.mc * 16; e += kSubThreads) {
                const int tok = e >> 4, oc = e & 15;
                const int rlo = (oc >> 3) * 16 + (oc & 7);
                const int c = jt * 16 + oc;
                float lo = sum_red(tok * 32 + rlo), hi = sum_red(tok * 32 + rlo + 8);
                if (NORM) {
                    lo *= s_rstd[tok];
                    hi *= s_rstd[tok];
                }
                lo += s_poison[tok];
                hi += s_poison[tok];
                if (p.bias) {
                    lo += __half2float(p.bias[n0 + rlo]);
                    hi += __half2float(p.bias[n0 + rlo + 8]);
                }
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
            }
        } else {
            if (tp_mode == 2) {
                // partial sums of a row-parallel GEMM: pairs of rows as one tagged 8-byte word straight into every rank's
                // inbox (own slot too); the word's tag makes it valid on arrival, nothing else is published
                for (int e = stid; e < p.mc * 16; e += kSubThreads) {
                    const int tok = e >> 4, row = (e & 15) * 2;
                    float v0 = sum_red(tok * 32 + row), v1 = sum_red(tok * 32 + row + 1);
                    if (NORM) {
                        v0 *= s_rstd[tok];
                        v1 *= s_rstd[tok];
                    }
                    v0 += s_poison[tok];
                    v1 += s_poison[tok];
                    if (p.bias) {
                        v0 += __half2float(p.bias[n0 + row]);
                        v1 += __half2float(p.bias[n0 + row + 1]);
                    }
                    const __half2 h2 = __floats2half2_rn(v0, v1);
                    const size_t word = ((size_t)tok * p.N + n0 + row) >> 1;
                    for (int r = 0; r < tp_ws; ++r)
                        st_ll(tp->inbox[r] + tp_my_slot + word * 8, *reinterpret_cast<const uint32_t*>(&h2), tp_tag);
                }
            } else {
                for (int e = stid; e < p.mc * 32; e += kSubThreads) {
                    const int tok = e >> 5, row = e & 31;
                    float v = sum_red(tok * 32 + row);
                    if (NORM) v *= s_rstd[tok];
                    v += s_poison[tok];
                    if (p.bias) v += __half2float(p.bias[n0 + row]);
                    __half h = __float2half_rn(v);
                    if (p.epi == ZL_EPI_RESIDUAL)
                        h = __float2half_rn(__half2float(h) + __half2float(p.residual[(size_t)tok * p.N + n0 + row]));
                    p.y[(size_t)tok * p.N + n0 + row] = h;
                }
            }
        }
        if (S::kRedBufs == 1) sub_barrier(1 + sub, WARPS * 32);
        stamp();
    }
}

static int v3_num_sms() { return device_sm_count(); }

constexpr int kV3Budget = 231000;   // one CTA per SM (227 KB usable + 1 KB reserved)

template <int NT, bool NORM, int WARPS, int SUBS, int STAGES, int RT, bool PACK>
static cudaError_t launch_v3_t(const W4Params& p, int smem, bool pdl, cudaStream_t stream) {
    const int tiles = p.N / 32;
    const int want = (tiles + SUBS - 1) / SUBS;
    const int grid = want < v3_num_sms() ? want : v3_num_sms();
    if (p.tp_mode != 0) {
        // exchange variants exist for the 4-stage rings only (launch_w4_v3 routes tensor-parallel launches there)
        if constexpr (STAGES == 4 && RT == NT * 8) {
            if (p.tp_mode == 1)
                return launch(k_w4a16_v3<NT, NORM, WARPS, SUBS, STAGES, RT, PACK, 1>, dim3(grid), dim3(WARPS * SUBS * 32),
                              (size_t)smem, stream, pdl, p);
            return launch(k_w4a16_v3<NT, NORM, WARPS, SUBS, STAGES, RT, PACK, 2>, dim3(grid), dim3(WARPS * SUBS * 32),
                          (size_t)smem, stream, pdl, p);
        } else {
            return cudaErrorNotSupported;
        }
    }
    return launch(k_w4a16_v3<NT, NORM, WARPS, SUBS, STAGES, RT, PACK>, dim3(grid), dim3(WARPS * SUBS * 32), (size_t)smem, stream,
                  pdl, p);
}

template <int NT, int WARPS, int SUBS, int STAGES, int RT = NT * 8>
static bool v3_try(const W4Params& p, bool pdl, cudaStream_t stream, cudaError_t* err) {
    const int G = p.K / kW4GroupK;
    const int smem = V3Smem<NT, WARPS, SUBS, STAGES, RT>::kBytes + v3_stage_bytes(p.mc, p.K);
    if (G > 8 * WARPS * SUBS || smem > kV3Budget || p.mc > RT) return false;   // 8 = kMaxNg
    static const bool no_one = getenv("ZL_W4_NO_ONE") != nullptr;
    if (NT == 1 && RT == NT * 8 && p.mc <= 4 && !no_one) {
        *err = p.ln_w ? launch_v3_t<NT, true, WARPS, SUBS, STAGES, RT, NT == 1 && RT == NT * 8>(p, smem, pdl, stream)
                      : launch_v3_t<NT, false, WARPS, SUBS, STAGES, RT, NT == 1 && RT == NT * 8>(p, smem, pdl, stream);
        return true;
    }
    *err = p.ln_w ? launch_v3_t<NT, true, WARPS, SUBS, STAGES, RT, false>(p, smem, pdl, stream)
                  : launch_v3_t<NT, false, WARPS, SUBS, STAGES, RT, false>(p, smem, pdl, stream);
    return true;
}

static int v3_max_stages() {
    static int v = -1;
    if (v < 0) {
        // deeper rings only add HBM
        // queueing, so the 6-stage variants stay opt-in
        const char* e = getenv("ZL_W4_STAGES");
        v = e ? atoi(e) : 4;
    }
    return v;
}

static bool v3_is_tall(const W4Params& p) {
    static int force = -1;
    if (force < 0) {
        const char* e = getenv("ZL_W4_TALL");
        force = e ? atoi(e) : 0;
    }
    if (force == 1) return p.K / kW4GroupK >= 32;
    if (force == 2) return false;
    return p.N / 32 <= v3_num_sms() && p.K / kW4GroupK >= 32;
}

// returns false when the staged activations do not fit shared memory (caller falls back to the fp16 kernels)
bool launch_w4_v3(const W4Params& p, bool pdl, cudaStream_t stream, cudaError_t* err) {
    const bool tall = v3_is_tall(p);
    if (p.tp_mode != 0) {   // fused tensor-parallel exchange: 4-stage variants
        if (p.mc <= 8) {
            if (tall && v3_try<1, 16, 1, 4>(p, pdl, stream, err)) return true;
            return v3_try<1, 8, 2, 4>(p, pdl, stream, err);
        }
        if (p.mc <= 16) {
            if (tall && v3_try<2, 16, 1, 4>(p, pdl, stream, err)) return true;
            return v3_try<2, 8, 2, 4>(p, pdl, stream, err);
        }
        return false;
    }
    if (p.mc <= 2) {   // deepest ring that fits (reduction buffers shrunk to 2 token rows)
        const int ms = v3_max_stages();
        if (tall) {
            if (ms >= 6 && v3_try<1, 16, 1, 6, 2>(p, pdl, stream, err)) return true;
            if (ms >= 5 && v3_try<1, 16, 1, 5, 2>(p, pdl, stream, err)) return true;
        } else {
            if (ms >= 6 && v3_try<1, 8, 2, 6, 2>(p, pdl, stream, err)) return true;
        }
    }
    if (p.mc <= 8) {
        if (tall && v3_try<1, 16, 1, 4>(p, pdl, stream, err)) return true;
        if (v3_try<1, 8, 2, 5>(p, pdl, stream, err)) return true;
        return v3_try<1, 8, 2, 4>(p, pdl, stream, err);
    }
    if (p.mc <= 16) {
        if (tall && v3_try<2, 16, 1, 4>(p, pdl, stream, err)) return true;
        return v3_try<2, 8, 2, 4>(p, pdl, stream, err);
    }
    return false;
}

bool w4_v3_fits(int mc, int N, int K) {
    const int G = K / kW4GroupK;
    if (G > 8 * 16) return false;
    const int stage = v3_stage_bytes(mc, K);
    if (mc <= 8) return V3Smem<1, 8, 2, 4>::kBytes + stage <= kV3Budget;
    if (mc <= 16) return V3Smem<2, 8, 2, 4>::kBytes + stage <= kV3Budget;
    (void)N;
    return false;
}

cudaError_t prepare_w4_v3() {
    cudaError_t e;
#define ZL_SET(NT, NORM, W, SB, ST)                                                                            \
    e = cudaFuncSetAttribute(k_w4a16_v3<NT, NORM, W, SB, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize,      \
                             kV3Budget);                                                                        \
    if (e != cudaSuccess) return e;
#define ZL_SET1(NORM, W, SB, ST)                                                                               \
    e = cudaFuncSetAttribute(k_w4a16_v3<1, NORM, W, SB, ST, 8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                             kV3Budget);                                                                        \
    if (e != cudaSuccess) return e;
    ZL_SET1(false, 8, 2, 5) ZL_SET1(true, 8, 2, 5) ZL_SET1(false, 8, 2, 4) ZL_SET1(true, 8, 2, 4)
    ZL_SET1(false, 16, 1, 4) ZL_SET1(true, 16, 1, 4)
#undef ZL_SET1
#define ZL_SET2(NORM, W, SB, ST)                                                                               \
    e = cudaFuncSetAttribute(k_w4a16_v3<1, NORM, W, SB, ST, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize,    \
                             kV3Budget);                                                                        \
    if (e != cudaSuccess) return e;
    ZL_SET2(false, 16, 1, 6) ZL_SET2(true, 16, 1, 6) ZL_SET2(false, 16, 1, 5) ZL_SET2(true, 16, 1, 5)
    ZL_SET2(false, 8, 2, 6) ZL_SET2(true, 8, 2, 6)
#undef ZL_SET2
    ZL_SET(1, false, 8, 2, 5) ZL_SET(1, true, 8, 2, 5) ZL_SET(1, false, 8, 2, 4) ZL_SET(1, true, 8, 2, 4)
    ZL_SET(1, false, 16, 1, 4) ZL_SET(1, true, 16, 1, 4)
    ZL_SET(2, false, 8, 2, 4) ZL_SET(2, true, 8, 2, 4) ZL_SET(2, false, 16, 1, 4) ZL_SET(2, true, 16, 1, 4)
#undef ZL_SET
#define ZL_SETX(NT, NORM, W, SB, PK)                                                                            \
    e = cudaFuncSetAttribute(k_w4a16_v3<NT, NORM, W, SB, 4, NT * 8, PK, 1>,                                     \
                             cudaFuncAttributeMaxDynamicSharedMemorySize, kV3Budget);                           \
    if (e != cudaSuccess) return e;                                                                             \
    e = cudaFuncSetAttribute(k_w4a16_v3<NT, NORM, W, SB, 4, NT * 8, PK, 2>,                                     \
                             cudaFuncAttributeMaxDynamicSharedMemorySize, kV3Budget);                           \
    if (e != cudaSuccess) return e;
    ZL_SETX(1, false, 8, 2, false) ZL_SETX(1, true, 8, 2, false) ZL_SETX(1, false, 16, 1, false) ZL_SETX(1, true, 16, 1, false)
    ZL_SETX(1, false, 8, 2, true) ZL_SETX(1, true, 8, 2, true) ZL_SETX(1, false, 16, 1, true) ZL_SETX(1, true, 16, 1, true)
    ZL_SETX(2, false, 8, 2, false) ZL_SETX(2, true, 8, 2, false) ZL_SETX(2, false, 16, 1, false) ZL_SETX(2, true, 16, 1, false)
#undef ZL_SETX
    return cudaSuccess;
}

}  // namespace zl
