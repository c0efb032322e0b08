// Causal variable-length attention over per-task KV caches: every row of a joined step -- prompt chunks and decode rows
// of different tasks -- in one launch.
//
// Stands in for Attention::dynamic_batch_forward over a chunked-prefill step that joins encode and search tokens
// (reference src/nn/attention/attention.cpp:924-961, scheduled by SearcherImplV1::join_forward,
// src/generator/batch_generator.cpp:1337-1422) with the contiguous-prefix causal mask of beam_size 1.  No mask is
// materialised: rows come in segments {task, row0, pos0, n} -- rows row0 .. row0 + n - 1 hold positions pos0 ..
// pos0 + n - 1 of `task` -- and the row at position p attends keys 0 ..= p of its task's BSHD cache.
//
// One CTA = (tile of up to QT consecutive query rows of one segment, kv head (its q heads, at most 64 per group), key
// split).  The tile's query rows x the group's q heads are the MMA rows (row qi * heads + h, 16 per warp), so every K/V
// byte staged in shared memory feeds the whole GQA group and every query row of the tile.  K/V tiles of 64 keys are
// double-buffered with cp.async (keys at or past the tile's last position + 1 are zero-filled, never read); S = Q.K^T and
// O += P.V run on mma.sync m16n8k16 with fp32 accumulate; softmax is online in fp32 (max seeded -1e20, the reference's
// 1e-20 added to the sum), and the P.V operand is encoded by attn_pack_p (fp16: p * 2^10 in fp16; bf16: hi + lo).
// Key tiles past the tile's last position are never visited, and only tiles that reach past its first position are
// masked per element.
//
// Batch invariance: split s always covers keys [512 s, 512 (s + 1)), whatever the launch holds.  A row's splits, and so
// its output bits, depend only on its q, its task's cache and its position.  A split holding none of a row's keys writes
// the empty partial (max -1e20, sum 1e-20, o = 0), which k_attn_combine weighs by exactly 0.
#include "attn_common.cuh"

namespace zl {

constexpr int kVaThreads = 128;
constexpr int kVaWarps = kVaThreads / 32;
constexpr int kVaMmaRows = 16 * kVaWarps;   // MMA rows of one CTA: query rows x q heads
constexpr int kVaMaxTileRows = 16;          // query rows of one tile
constexpr int kVaKeyTile = 64;              // keys per shared-memory stage
constexpr int kVaSplitKeys = 512;           // keys per split (fixed: batch invariance)

template <int D>
constexpr int va_smem_bytes() {
    return 2 * 2 * kVaKeyTile * D * 2;   // {K, V} x 2 stages x 64 keys x D x 16 bit
}

// element offset of 16-byte chunk c of key row r in a (64, D) stage: chunks XOR-swizzled by r & 7, so that the 8 rows an
// ldmatrix phase reads at one logical chunk sit in 8 different bank groups
template <int D>
__device__ __forceinline__ int va_off(int r, int c) {
    return r * D + ((c ^ (r & 7)) << 3);
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
template <typename T, int D>
__global__ void __launch_bounds__(kVaThreads)
k_varlen_attn(const T* __restrict__ q, const int4* __restrict__ seg, int nseg, T* const* __restrict__ k_addrs,
              T* const* __restrict__ v_addrs, float scale, T* __restrict__ out, float* __restrict__ part_o,
              float* __restrict__ part_m, float* __restrict__ part_l, int num_heads, int num_kv_heads, int m_query,
              int group_heads, int tile_rows, int num_splits) {
    constexpr int DC = D / 8;    // 16-byte chunks of a key row = n-tiles of O
    constexpr int NK = D / 16;   // k-steps of S = Q.K^T
    constexpr int NS = kVaKeyTile / 8;   // n-tiles of S
    constexpr bool kHalf = std::is_same<T, __half>::value;
    extern __shared__ __align__(128) uint8_t va_smem[];
    T* sk = reinterpret_cast<T*>(va_smem);   // [2][64][D]
    T* sv = sk + 2 * kVaKeyTile * D;         // [2][64][D]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    pdl_trigger();
    pdl_wait();

    // this CTA's tile: the blockIdx.x-th tile_rows-row tile of the segments in order; surplus CTAs exit
    int tile = blockIdx.x, si = 0;
    int4 sg = make_int4(0, 0, 0, 0);
    for (; si < nseg; ++si) {
        sg = seg[si];
        const int nt = sg.w > 0 ? (sg.w + tile_rows - 1) / tile_rows : 0;
        if (tile < nt) break;
        tile -= nt;
    }
    if (si >= nseg) return;
    const int task = sg.x, row0 = sg.y + tile * tile_rows, pos_first = sg.z + tile * tile_rows;
    const int nq = min(tile_rows, sg.w - tile * tile_rows);
    const int hgroups = (m_query + group_heads - 1) / group_heads;
    const int hk = blockIdx.y / hgroups, hg = blockIdx.y % hgroups;
    const int mh = min(group_heads, m_query - hg * group_heads);
    const int head0 = hk * m_query + hg * group_heads;
    const int nrows = nq * mh;
    const int split = blockIdx.z;
    const int kb0 = split * kVaSplitKeys;
    const int k_end = min(pos_first + nq, kb0 + kVaSplitKeys);   // keys [kb0, k_end) are read, none past k_end
    const int ntiles = k_end > kb0 ? (k_end - kb0 + kVaKeyTile - 1) / kVaKeyTile : 0;

    // MMA rows of this lane: ra = 16 warp + g and rb = ra + 8 -> (query row r / mh, head r % mh)
    const bool active = warp * 16 < nrows;
    int qi_r[2] = {0, 0}, h_r[2] = {0, 0}, pos_r[2] = {-1, -1};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int r = warp * 16 + g + 8 * i;
        if (r < nrows) {
            qi_r[i] = r / mh;
            h_r[i] = r % mh;
            pos_r[i] = pos_first + qi_r[i];
        }
    }
    uint32_t qf[NK][4];
    {
        const T* qa = q + ((size_t)(row0 + qi_r[0]) * num_heads + head0 + h_r[0]) * D + 2 * t;
        const T* qb = q + ((size_t)(row0 + qi_r[1]) * num_heads + head0 + h_r[1]) * D + 2 * t;
        const bool va = pos_r[0] >= 0, vb = pos_r[1] >= 0;
#pragma unroll
        for (int kk = 0; kk < NK; ++kk) {
            qf[kk][0] = va ? __ldcg(reinterpret_cast<const unsigned*>(qa + kk * 16)) : 0u;
            qf[kk][1] = vb ? __ldcg(reinterpret_cast<const unsigned*>(qb + kk * 16)) : 0u;
            qf[kk][2] = va ? __ldcg(reinterpret_cast<const unsigned*>(qa + kk * 16 + 8)) : 0u;
            qf[kk][3] = vb ? __ldcg(reinterpret_cast<const unsigned*>(qb + kk * 16 + 8)) : 0u;
        }
    }

    const size_t stride = (size_t)num_kv_heads * D;
    const T* kbase = k_addrs[task] + (size_t)hk * D;
    const T* vbase = v_addrs[task] + (size_t)hk * D;
    auto load_stage = [&](int it) {
        const int kb = kb0 + it * kVaKeyTile;
        T* dk = sk + (it & 1) * kVaKeyTile * D;
        T* dv = sv + (it & 1) * kVaKeyTile * D;
        for (int i = tid; i < kVaKeyTile * DC; i += kVaThreads) {
            const int r = i / DC, c = i % DC;
            const bool ok = kb + r < k_end;
            const size_t off = ok ? (size_t)(kb + r) * stride + c * 8 : 0;
            cp_async16(smem_u32(dk + va_off<D>(r, c)), kbase + off, ok ? 16 : 0);
            cp_async16(smem_u32(dv + va_off<D>(r, c)), vbase + off, ok ? 16 : 0);
        }
        cp_async_commit();
    };

    float m_r[2] = {-1e20f, -1e20f}, l_r[2] = {0.f, 0.f};
    float o[DC][4];
#pragma unroll
    for (int j = 0; j < DC; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;

    if (ntiles > 0) load_stage(0);
    for (int it = 0; it < ntiles; ++it) {
        if (it + 1 < ntiles) {
            load_stage(it + 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (active) {
            const uint32_t tk = smem_u32(sk + (it & 1) * kVaKeyTile * D);
            const uint32_t tv = smem_u32(sv + (it & 1) * kVaKeyTile * D);
            const int mat = lane >> 3, mr = lane & 7;
            // ---- S = Q.K^T: B = K rows (n = key, k = dim), two n-tiles per ldmatrix.x4 ----
            float s[NS][4];
#pragma unroll
            for (int j = 0; j < NS; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
            for (int kk = 0; kk < NK; ++kk) {
#pragma unroll
                for (int jp = 0; jp < NS / 2; ++jp) {
                    const int r = 16 * jp + (mat >> 1) * 8 + mr, c = 2 * kk + (mat & 1);
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4(tk + 2 * va_off<D>(r, c), b0, b1, b2, b3);
                    mma_attn<T>(s[2 * jp], qf[kk], b0, b1);
                    mma_attn<T>(s[2 * jp + 1], qf[kk], b2, b3);
                }
            }
            // ---- causal mask (tiles reaching past the tile's first position) and online softmax ----
            const int kb = kb0 + it * kVaKeyTile;
            const bool diag = kb + kVaKeyTile - 1 > pos_first;
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int j = 0; j < NS; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int i = e >> 1;
                    float v = s[j][e] * scale;
                    if (diag && kb + 8 * j + 2 * t + (e & 1) > pos_r[i]) v = -INFINITY;
                    s[j][e] = v;
                    mx[i] = fmaxf(mx[i], v);
                }
            float alpha[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float mn = fmaxf(m_r[i], quad_max(mx[i]));
                alpha[i] = expf(m_r[i] - mn);
                m_r[i] = mn;
            }
            float ps[2] = {0.f, 0.f};
#pragma unroll
            for (int j = 0; j < NS; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float p = expf(s[j][e] - m_r[e >> 1]);
                    s[j][e] = p;
                    ps[e >> 1] += p;
                }
#pragma unroll
            for (int i = 0; i < 2; ++i) l_r[i] = l_r[i] * alpha[i] + ps[i];
#pragma unroll
            for (int j = 0; j < DC; ++j) {
                o[j][0] *= alpha[0];
                o[j][1] *= alpha[0];
                o[j][2] *= alpha[1];
                o[j][3] *= alpha[1];
            }
            // ---- O += P.V: A = P from the S accumulators, B = V rows (k = key, n = dim) via ldmatrix.trans ----
#pragma unroll
            for (int kk = 0; kk < kVaKeyTile / 16; ++kk) {
                uint32_t af[4], al[4];
                attn_pack_p<T>(s[2 * kk][0], s[2 * kk][1], af[0], al[0]);
                attn_pack_p<T>(s[2 * kk][2], s[2 * kk][3], af[1], al[1]);
                attn_pack_p<T>(s[2 * kk + 1][0], s[2 * kk + 1][1], af[2], al[2]);
                attn_pack_p<T>(s[2 * kk + 1][2], s[2 * kk + 1][3], af[3], al[3]);
#pragma unroll
                for (int jp = 0; jp < DC / 2; ++jp) {
                    const int r = 16 * kk + (mat & 1) * 8 + mr, c = 2 * jp + (mat >> 1);
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4_t(tv + 2 * va_off<D>(r, c), b0, b1, b2, b3);
                    mma_attn<T>(o[2 * jp], af, b0, b1);
                    mma_attn<T>(o[2 * jp + 1], af, b2, b3);
                    if constexpr (!kHalf) {
                        mma_attn<T>(o[2 * jp], al, b0, b1);
                        mma_attn<T>(o[2 * jp + 1], al, b2, b3);
                    }
                }
            }
        }
        __syncthreads();   // the stage just read is refilled by the next iteration's load
    }

    if (!active) return;
    const float sc = kHalf ? (1.f / 1024.f) : 1.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float l = quad_sum(l_r[i]) + 1e-20f;
        if (pos_r[i] < 0) continue;
        const size_t vh = (size_t)(row0 + qi_r[i]) * num_heads + head0 + h_r[i];
        if (num_splits == 1) {
            T* dst = out + vh * D + 2 * t;
#pragma unroll
            for (int j = 0; j < DC; ++j) {
                dst[8 * j] = from_f32<T>(o[j][2 * i] * sc / l);
                dst[8 * j + 1] = from_f32<T>(o[j][2 * i + 1] * sc / l);
            }
        } else {
            float* dst = part_o + (vh * num_splits + split) * D + 2 * t;
#pragma unroll
            for (int j = 0; j < DC; ++j)
                *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[j][2 * i] * sc / l, o[j][2 * i + 1] * sc / l);
            if (t == 0) {
                part_m[vh * num_splits + split] = m_r[i];
                part_l[vh * num_splits + split] = l;
            }
        }
    }
}

// q heads of one CTA group and query rows of one tile: at most 64 MMA rows per CTA
inline int va_group_heads(int m_query) { return m_query < kVaMmaRows ? m_query : kVaMmaRows; }
inline int va_tile_rows(int group_heads) {
    const int r = kVaMmaRows / group_heads;
    return r < 1 ? 1 : (r > kVaMaxTileRows ? kVaMaxTileRows : r);
}

}  // namespace zl

using namespace zl;

extern "C" size_t zl_varlen_attention_workspace_bytes(int rows, int nseg, int num_heads, int dim_head, int max_keys) {
    if (rows <= 0 || nseg <= 0 || nseg > rows || num_heads <= 0 || dim_head <= 0 || max_keys <= 0) return 0;
    const int splits = cdiv(max_keys, kVaSplitKeys);
    return splits > 1 ? attn_parts_bytes((size_t)rows * num_heads, splits, dim_head) : 0;
}

extern "C" int zl_varlen_attention(const void* q, const int32_t* seg, int nseg, int rows, void* const* k_addrs,
                                   void* const* v_addrs, float scale, int max_keys, void* out, int num_heads,
                                   int num_kv_heads, int dim_head, void* ws, size_t ws_bytes, int dtype, int pdl,
                                   zl_stream_t stream) {
    ZL_CHECK_ARG(q && seg && k_addrs && v_addrs && out);
    ZL_CHECK_ARG(nseg > 0 && rows > 0 && nseg <= rows && max_keys > 0);
    ZL_CHECK_ARG(num_heads > 0 && num_kv_heads > 0 && num_heads % num_kv_heads == 0);
    ZL_CHECK_SUPPORTED(dim_head == 64 || dim_head == 128);
    ZL_CHECK_SUPPORTED(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_ARG(reinterpret_cast<uintptr_t>(seg) % 16 == 0);
    const int splits = cdiv(max_keys, kVaSplitKeys);
    ZL_CHECK_SUPPORTED(splits <= 65535);
    const size_t vheads = (size_t)rows * num_heads;
    if (splits > 1) ZL_CHECK_ARG(ws != nullptr && ws_bytes >= attn_parts_bytes(vheads, splits, dim_head));
    const AttnParts part = attn_parts(ws, vheads, splits, dim_head);
    const int m_query = num_heads / num_kv_heads;
    const int gh = va_group_heads(m_query), qt = va_tile_rows(gh);
    const dim3 grid(cdiv(rows, qt) + nseg, num_kv_heads * cdiv(m_query, gh), splits);
    cudaStream_t st = (cudaStream_t)stream;
#define ZL_VA_LAUNCH(TT, DD)                                                                                          \
    {                                                                                                                 \
        ZL_CHECK_CUDA((attn_smem_opt_in<k_varlen_attn<TT, DD>>(va_smem_bytes<DD>())));                                \
        ZL_CHECK_CUDA(launch(k_varlen_attn<TT, DD>, grid, dim3(kVaThreads), (size_t)va_smem_bytes<DD>(), st, pdl != 0, \
                             (const TT*)q, (const int4*)seg, nseg, (TT* const*)k_addrs, (TT* const*)v_addrs, scale,    \
                             (TT*)out, part.o, part.m, part.l, num_heads, num_kv_heads, m_query, gh, qt, splits));    \
        ZL_CHECK_CUDA(launch_attn_combine(part, vheads, DD, (TT*)out, splits, st, pdl != 0));                         \
    }
    if (dtype == ZL_F16) {
        if (dim_head == 128) ZL_VA_LAUNCH(__half, 128) else ZL_VA_LAUNCH(__half, 64)
    } else {
        if (dim_head == 128) ZL_VA_LAUNCH(__nv_bfloat16, 128) else ZL_VA_LAUNCH(__nv_bfloat16, 64)
    }
#undef ZL_VA_LAUNCH
    return ZL_OK;
}
