// MLA (multi-head latent attention) decode attention over per-task latent caches, on wgmma.
//
// Replaces nn::multi_query_attention_rag_buffer with dim_head == 576 and a 512-wide output, the reference's fused MLA
// search path (src/nn/attention/multi_head_latent_attention.cpp:1053-1068 -> attention_kernel.cu:1281-1284,
// 1347-1348, 1390-1391, 1429-1435), and the three-launch attn_by_gemm it falls back to (:834-874).  A task's cache holds
// one 576-element latent row per token: the whole row is every query head's key, its first 512 elements its value.
//
// One CTA = (key split, tile of up to 64 query rows, task).  The task's len_q x H (query, head) pairs are packed into the
// tile's rows, so every latent byte staged in shared memory feeds all of them: the cache is read from HBM once per row
// tile, not once per head.  Two consumer warpgroups each own 256 of the 512 output columns (64 x 256 fp32
// accumulators per warpgroup):
//   * S = Q.K^T runs as wgmma m64n64k16 with both operands in shared memory (Q tile 64 x 576, K tile 64 keys x 576,
//     128-byte-swizzled, K-major).  Both warpgroups compute the same S, so their softmax statistics agree bit for bit
//     and no shared-memory exchange is needed;
//   * softmax is online in fp32 (max seeded -1e20, the reference's 1e-20 added to the sum, attention_kernel.cu:434-489);
//   * O += P.V runs as wgmma m64n256k16 with P from registers (the S accumulator layout is the A fragment layout) and V
//     = the first 512 columns of the SAME shared-memory K tile, read as a transposed (MN-major) B operand.
// K tiles of 64 keys are double-buffered with cp.async 16-byte copies written straight into the swizzled layout: the
// per-task caches are reached through a device pointer table, which a host-encoded tensor map could not follow without a
// host sync.  Keys past the split's end are zero-filled, never read, so stale or NaN cache rows cannot reach P.V.
// P is carried in 16 bits: fp16 models as p * 2^10 in fp16 (11 significant bits), bf16 models as bf16 (8 bits; a
// hi + lo pair would double the P.V MMAs that bound H = 128).  Key splits are merged by k_attn_combine in a fixed order.
#include "attn_common.cuh"
#include "tc_common.cuh"

namespace zl {

constexpr int kMlaD = 576;                       // latent row: kv_lora_rank 512 + rope 64
constexpr int kMlaDv = 512;                      // value / output width
constexpr int kMlaRows = 64;                     // query rows (query x head pairs) of one CTA
constexpr int kMlaKeys = 64;                     // keys per shared-memory stage
constexpr int kMlaThreads = 256;                 // two consumer warpgroups
constexpr int kMlaChunks = kMlaD / 8;            // 16-byte chunks of a row
constexpr int kMlaBlk = 64 * 128;                // one 64-column block of a 64-row tile: 64 rows x 128 B
constexpr int kMlaTile = kMlaRows * kMlaD * 2;   // 73,728 B: the Q tile and each K stage
constexpr int kMlaSmem = 3 * kMlaTile + 1024;    // Q + two K stages + slack for the manual 1024-byte alignment
constexpr int kMlaMaxHeads = 128;
constexpr int kMlaMinSplitKeys = 256;            // a split covers at least this many keys
constexpr int kMlaMaxSplits = 64;

// byte offset of 16-byte chunk c of row r in a (64, 576) tile: nine 64-column blocks of 64 rows x 128 B, chunks
// XOR-swizzled by r & 7 (the SWIZZLE_128B pattern of wgmma descriptors; the tile is 1024-byte aligned)
__device__ __forceinline__ uint32_t mla_off(int r, int c) {
    return (uint32_t)((c >> 3) * kMlaBlk + r * 128 + (((c & 7) ^ (r & 7)) << 4));
}

// 128-byte-swizzle matrix descriptor: SBO = 1024 B between 8-row groups; LBO is unused for K-major operands (canonical
// value 16 B) and is the stride between 64-element column blocks for an MN-major operand
__device__ __forceinline__ uint64_t mla_desc(uint32_t saddr, uint32_t lbo) {
    uint64_t d = (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

#define MLA_ACC8(C, i) C(d[i]), C(d[i + 1]), C(d[i + 2]), C(d[i + 3]), C(d[i + 4]), C(d[i + 5]), C(d[i + 6]), C(d[i + 7])
#define MLA_D32 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"
#define MLA_D128 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}"
#define MLA_ACC32 MLA_ACC8("+f", 0), MLA_ACC8("+f", 8), MLA_ACC8("+f", 16), MLA_ACC8("+f", 24)
#define MLA_ACC128                                                                                                    \
    MLA_ACC8("+f", 0), MLA_ACC8("+f", 8), MLA_ACC8("+f", 16), MLA_ACC8("+f", 24), MLA_ACC8("+f", 32),                 \
        MLA_ACC8("+f", 40), MLA_ACC8("+f", 48), MLA_ACC8("+f", 56), MLA_ACC8("+f", 64), MLA_ACC8("+f", 72),           \
        MLA_ACC8("+f", 80), MLA_ACC8("+f", 88), MLA_ACC8("+f", 96), MLA_ACC8("+f", 104), MLA_ACC8("+f", 112),         \
        MLA_ACC8("+f", 120)

// S (64 x 64) (+)= A (64 x 16, K-major smem) . B (64 keys x 16, K-major smem)^T
template <bool BF>
__device__ __forceinline__ void mla_wg_qk(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    if constexpr (BF) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\nwgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " MLA_D32
                     ", %32, %33, p, 1, 1, 0, 0;\n}"
                     : MLA_ACC32 : "l"(adesc), "l"(bdesc), "r"(accum));
    } else {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\nwgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " MLA_D32
                     ", %32, %33, p, 1, 1, 0, 0;\n}"
                     : MLA_ACC32 : "l"(adesc), "l"(bdesc), "r"(accum));
    }
}
// O (64 x 256) += P (64 x 16 keys, registers) . V (16 keys x 256, MN-major smem: transposed B)
template <bool BF>
__device__ __forceinline__ void mla_wg_pv(float (&d)[128], const uint32_t (&a)[4], uint64_t bdesc) {
    if constexpr (BF) {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %133, 0;\nwgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " MLA_D128
                     ", {%128,%129,%130,%131}, %132, p, 1, 1, 1;\n}"
                     : MLA_ACC128 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1u));
    } else {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %133, 0;\nwgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " MLA_D128
                     ", {%128,%129,%130,%131}, %132, p, 1, 1, 1;\n}"
                     : MLA_ACC128 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1u));
    }
}
#undef MLA_ACC128
#undef MLA_ACC32
#undef MLA_D128
#undef MLA_D32
#undef MLA_ACC8

// grid (num_splits, row tiles, B), block kMlaThreads, dynamic shared memory kMlaSmem
template <typename T>
__global__ void __launch_bounds__(kMlaThreads, 1)
k_mla_decode_attn(const T* __restrict__ q, const int32_t* __restrict__ buf_lens, T* const* __restrict__ kv_addrs,
                  const int8_t* __restrict__ mask, float scale, T* __restrict__ out, float* __restrict__ part_o,
                  float* __restrict__ part_m, float* __restrict__ part_l, int len_q, int num_heads, int num_splits) {
    constexpr bool kHalf = std::is_same<T, __half>::value;
    extern __shared__ __align__(1024) uint8_t mla_smem_raw[];
    const uint32_t sq = smem_u32(mla_smem_raw) + ((1024u - (smem_u32(mla_smem_raw) & 1023u)) & 1023u);
    const uint32_t sk = sq + kMlaTile;   // stage s at sk + s * kMlaTile

    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int split = blockIdx.x, b = blockIdx.z;
    const int task_rows = len_q * num_heads;
    const int row0 = blockIdx.y * kMlaRows;
    const int nrows = min(kMlaRows, task_rows - row0);
    pdl_trigger();
    pdl_wait();

    const int len_buf = buf_lens[b];
    const int chunk = cdiv(cdiv(len_buf, num_splits), kMlaKeys) * kMlaKeys;
    const int k0 = split * chunk;
    const int k1 = min(len_buf, k0 + chunk);
    const int ntiles = k1 > k0 ? cdiv(k1 - k0, kMlaKeys) : 0;

    // this thread's accumulator rows: 16 warp + g and + 8 of the tile
    int r_row[2];
    const int8_t* mrow[2] = {nullptr, nullptr};
    const size_t len_off = mask ? attn_keys_before(buf_lens, b) : 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        r_row[i] = warp * 16 + g + 8 * i;
        const int qi = r_row[i] < nrows ? (row0 + r_row[i]) / num_heads : 0;
        if (mask) mrow[i] = mask + (size_t)len_q * len_off + (size_t)qi * len_buf;
    }

    const T* qbase = q + ((size_t)b * task_rows + row0) * kMlaD;
    const T* kvbase = kv_addrs[b];
    auto load_stage = [&](int it) {
        const int kb = k0 + it * kMlaKeys;
        const uint32_t dst = sk + (it & 1) * kMlaTile;
        for (int i = tid; i < kMlaKeys * kMlaChunks; i += kMlaThreads) {
            const int r = i / kMlaChunks, c = i % kMlaChunks;
            const bool ok = kb + r < k1;
            cp_async16(dst + mla_off(r, c), kvbase + (ok ? (size_t)(kb + r) * kMlaD + c * 8 : 0), ok ? 16 : 0);
        }
        cp_async_commit();
    };

    float o[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) o[j] = 0.f;
    float m_r[2] = {-1e20f, -1e20f}, l_r[2] = {0.f, 0.f};

    if (ntiles > 0) {
        for (int i = tid; i < kMlaRows * kMlaChunks; i += kMlaThreads) {
            const int r = i / kMlaChunks, c = i % kMlaChunks;
            const bool ok = r < nrows;
            cp_async16(sq + mla_off(r, c), qbase + (ok ? (size_t)r * kMlaD + c * 8 : 0), ok ? 16 : 0);
        }
        load_stage(0);
    }
    for (int it = 0; it < ntiles; ++it) {
        if (it + 1 < ntiles) {
            load_stage(it + 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        // cp.async wrote through the generic proxy; wgmma reads through the async proxy
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        const uint32_t kt = sk + (it & 1) * kMlaTile;

        // ---- S = Q.K^T (36 k-steps of 16 over the 576-wide rows) ----
        float s[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) s[j] = 0.f;
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < kMlaD / 16; ++kk) {
            const uint32_t off = (kk >> 2) * kMlaBlk + (kk & 3) * 32;
            mla_wg_qk<!kHalf>(s, mla_desc(sq + off, 16), mla_desc(kt + off, 16), kk > 0 ? 1u : 0u);
        }
        wg_commit();
        wg_wait_all();

        // ---- mask (keys past the split's end, and the optional mask) and online softmax ----
        const int kb = k0 + it * kMlaKeys;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i = e >> 1, key = kb + 8 * j + 2 * t + (e & 1);
                const bool ok = key < k1 && (mrow[i] == nullptr || mrow[i][key] != 0);
                const float v = ok ? s[4 * j + e] * scale : -INFINITY;
                s[4 * j + e] = v;
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
        for (int j = 0; j < 32; ++j) {
            const float p = expf(s[j] - m_r[(j >> 1) & 1]);
            s[j] = p;
            ps[(j >> 1) & 1] += p;
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) l_r[i] = l_r[i] * alpha[i] + ps[i];
#pragma unroll
        for (int j = 0; j < 128; ++j) o[j] *= alpha[(j >> 1) & 1];

        // ---- O += P.V: k-step kk covers keys 16 kk .. 16 kk + 15; this warpgroup's columns start at block 4 wg ----
        uint32_t a[4][4], lo;   // lo is unused: P.V runs on the hi word alone
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int r = 0; r < 4; ++r) attn_pack_p<T>(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1], a[kk][r], lo);
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) mla_wg_pv<!kHalf>(o, a[kk], mla_desc(kt + wg * 4 * kMlaBlk + kk * 2048, kMlaBlk));
        wg_commit();
        wg_wait_all();
        __syncthreads();   // the stage just read is refilled by the next iteration's load
    }

    const float sc = kHalf ? (1.f / 1024.f) : 1.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float l = quad_sum(l_r[i]) + 1e-20f;
        if (r_row[i] >= nrows) continue;
        const size_t vh = (size_t)b * task_rows + row0 + r_row[i];
        const int col0 = wg * 256 + 2 * t;
        if (num_splits == 1) {
            T* dst = out + vh * kMlaDv + col0;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const float x = o[4 * j + 2 * i] * sc / l, y = o[4 * j + 2 * i + 1] * sc / l;
                if constexpr (kHalf) {
                    *reinterpret_cast<__half2*>(dst + 8 * j) = __floats2half2_rn(x, y);
                } else {
                    *reinterpret_cast<__nv_bfloat162*>(dst + 8 * j) = __floats2bfloat162_rn(x, y);
                }
            }
        } else {
            float* dst = part_o + (vh * num_splits + split) * kMlaDv + col0;
#pragma unroll
            for (int j = 0; j < 32; ++j)
                *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[4 * j + 2 * i] * sc / l, o[4 * j + 2 * i + 1] * sc / l);
            if (wg == 0 && t == 0) {
                part_m[vh * num_splits + split] = m_r[i];
                part_l[vh * num_splits + split] = l;
            }
        }
    }
}

// upper bound of the split count for a given max_len_buf: the workspace is sized by it
inline int mla_max_splits(int max_len_buf) {
    const int s = cdiv(max_len_buf, kMlaMinSplitKeys);
    return s < 1 ? 1 : (s > kMlaMaxSplits ? kMlaMaxSplits : s);
}

// one CTA per SM (the tiles take 216 KiB of shared memory): split keys only while B x row tiles leaves SMs idle, and
// never into more CTAs than one wave
inline int mla_num_splits(int B, int row_tiles, int max_len_buf) {
    const long long base = (long long)B * row_tiles;
    const long long fit = device_sm_count() / base;
    const int s = mla_max_splits(max_len_buf);
    return fit < 1 ? 1 : (fit < s ? (int)fit : s);
}

}  // namespace zl

using namespace zl;

extern "C" size_t zl_mla_decode_attention_workspace_bytes(int B, int len_q, int num_heads, int max_len_buf) {
    if (B <= 0 || len_q <= 0 || num_heads <= 0 || max_len_buf <= 0) return 0;
    const int s = mla_max_splits(max_len_buf);
    return s > 1 ? attn_parts_bytes((size_t)B * len_q * num_heads, s, kMlaDv) : 0;
}

extern "C" int zl_mla_decode_attention(const void* q, const int32_t* buf_lens, void* const* kv_addrs, const int8_t* mask,
                                       float scale, int max_len_buf, void* out, int B, int len_q, int num_heads,
                                       void* workspace, size_t workspace_bytes, int dtype, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(q && buf_lens && kv_addrs && out && B > 0 && len_q > 0 && num_heads > 0 && max_len_buf > 0);
    ZL_CHECK_SUPPORTED(num_heads <= kMlaMaxHeads);
    ZL_CHECK_SUPPORTED(dtype == ZL_F16 || dtype == ZL_BF16);
    ZL_CHECK_SUPPORTED(B <= 65535 && (long long)len_q * num_heads <= 65535LL * kMlaRows);
    const size_t need = zl_mla_decode_attention_workspace_bytes(B, len_q, num_heads, max_len_buf);
    ZL_CHECK_ARG(need == 0 || (workspace != nullptr && workspace_bytes >= need));
    const int row_tiles = cdiv(len_q * num_heads, kMlaRows);
    const int splits = mla_num_splits(B, row_tiles, max_len_buf);
    const size_t vheads = (size_t)B * len_q * num_heads;
    const AttnParts part = attn_parts(workspace, vheads, splits, kMlaDv);
    const dim3 grid(splits, row_tiles, B);
    cudaStream_t st = (cudaStream_t)stream;
#define ZL_MLA_LAUNCH(TT)                                                                                              \
    {                                                                                                                  \
        ZL_CHECK_CUDA(attn_smem_opt_in<k_mla_decode_attn<TT>>(kMlaSmem));                                             \
        ZL_CHECK_CUDA(launch(k_mla_decode_attn<TT>, grid, dim3(kMlaThreads), (size_t)kMlaSmem, st, pdl != 0,           \
                             (const TT*)q, buf_lens, (TT* const*)kv_addrs, mask, scale, (TT*)out, part.o, part.m,     \
                             part.l, len_q, num_heads, splits));                                                       \
        ZL_CHECK_CUDA(launch_attn_combine(part, vheads, kMlaDv, (TT*)out, splits, st, pdl != 0));                     \
    }
    if (dtype == ZL_F16) ZL_MLA_LAUNCH(__half) else ZL_MLA_LAUNCH(__nv_bfloat16)
#undef ZL_MLA_LAUNCH
    return ZL_OK;
}
