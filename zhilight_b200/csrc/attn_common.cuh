// Pieces shared by the attention kernels: k_decode_attn (decode_attn.cu), k_decode_attn_warp (decode_attn_warp.cuh),
// k_decode_attn_kv8 (decode_attn_kv8.cu), k_varlen_attn (varlen_attn.cu) and k_mla_decode_attn (mla_attn.cu).
//   * device: the per-type tensor-core MMA, cp.async, quad shuffles, the P.V A-operand encoding, the decode CTA work
//     item with its q fragment and output store, and k_attn_combine, which merges key splits;
//   * host: the decode split count, the split partials carved from a workspace, and the opt-in to large dynamic shared
//     memory on each device.
#pragma once
#include "common.cuh"

#include <type_traits>

namespace zl {

__host__ __device__ inline int attn_round16(int v) { return (v + 15) & ~15; }

template <typename T>
__device__ __forceinline__ void mma_attn(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma_attn<__half>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    mma_16816_f16(d, a, b0, b1, d);
}
template <>
__device__ __forceinline__ void mma_attn<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                                        uint32_t b1) {
    mma_16816_bf16(d, a, b0, b1, d);
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// reductions over the 4 lanes (t = 0..3) that hold one MMA accumulator row
__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// The P.V A operand of probabilities (x, y) (lower key first).  fp16 models carry p * 2^10 in fp16 (11 significant
// bits, no subnormals; the accumulators are scaled back by 2^-10); bf16 models carry p as bf16 hi + lo, two MMAs, so
// that the product keeps ~16 bits of p.  A caller that runs only the hi MMA ignores lo.
template <typename T>
__device__ __forceinline__ void attn_pack_p(float x, float y, uint32_t& hi, uint32_t& lo) {
    if constexpr (std::is_same<T, __half>::value) {
        const __half2 h = __floats2half2_rn(x * 1024.f, y * 1024.f);
        hi = *reinterpret_cast<const uint32_t*>(&h);
        lo = 0u;
    } else {
        const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
        const float2 f = __bfloat1622float2(h);
        const __nv_bfloat162 l = __floats2bfloat162_rn(x - f.x, y - f.y);
        hi = *reinterpret_cast<const uint32_t*>(&h);
        lo = *reinterpret_cast<const uint32_t*>(&l);
    }
}

// The ragged mask concatenates one (len_q, len_buf) int8 block per task: task b's block starts at row len_q times the
// keys of the tasks before it.
__device__ __forceinline__ size_t attn_keys_before(const int32_t* buf_lens, int b) {
    size_t len_off = 0;
    for (int j = 0; j < b; ++j) len_off += buf_lens[j];
    return len_off;
}

// ---------------------------------------------------------------------------------------------------------------------
// Decode attention (k_decode_attn, k_decode_attn_warp, k_decode_attn_kv8): grid (key split, kv head x head group,
// task x query).  A head group is up to 8 of a kv head's m_query q heads; a split covers chunk = round16(cdiv(len_buf,
// num_splits)) keys of the task.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kAttnThreads = 128;                // k_decode_attn, k_decode_attn_kv8
constexpr int kAttnWarps = kAttnThreads / 32;
constexpr int kAttnMaxRange = 1024;              // keys per CTA; logits live in shared memory
constexpr int kAttnRowStride = kAttnMaxRange + 4;
constexpr int kAttnMaxSplits = 64;
// keys per split in the latency regime (few CTAs of work), where zl_decode_attention runs the warp kernel
constexpr int kShortRange = 256;

struct DecodeAttnItem {
    int split, hk, bq, b;     // key split, kv head, task x query and task
    int mq, head0;            // q heads of the group (<= 8) and the first one's index
    int qi, len_buf, k0, k1;  // query, the task's keys, and the split's keys [k0, k1) (empty past len_buf)

    // the query's row of the ragged mask, or nullptr for no mask.  Kernels ask for it after loading their cache
    // pointers: ahead of those loads it costs k_decode_attn<bf16, 128> two registers.
    __device__ __forceinline__ const int8_t* mask_row(const int8_t* mask, const int32_t* buf_lens, int len_q) const {
        return mask ? mask + (size_t)len_q * attn_keys_before(buf_lens, b) + (size_t)qi * len_buf : nullptr;
    }
};

// The prologue of a decode-attention CTA: its work item from blockIdx, the PDL trigger and wait, and then the split's
// keys, which read buf_lens.  The index arithmetic stays ahead of the wait, where it overlaps the
// predecessor kernel.
__device__ __forceinline__ DecodeAttnItem decode_attn_prologue(const int32_t* buf_lens, int len_q, int m_query,
                                                               int num_splits) {
    DecodeAttnItem cta;
    const int hgroups = (m_query + 7) / 8;
    cta.split = blockIdx.x;
    cta.hk = blockIdx.y / hgroups;
    const int hg = blockIdx.y % hgroups;
    cta.bq = blockIdx.z;
    cta.b = cta.bq / len_q;
    cta.qi = cta.bq % len_q;
    cta.mq = min(8, m_query - hg * 8);
    cta.head0 = cta.hk * m_query + hg * 8;

    pdl_trigger();
    pdl_wait();

    cta.len_buf = buf_lens[cta.b];
    const int chunk = attn_round16((cta.len_buf + num_splits - 1) / num_splits);
    cta.k0 = cta.split * chunk;
    cta.k1 = min(cta.len_buf, cta.k0 + chunk);
    return cta;
}

// lane (g, t)'s q fragment, the B operand of S = K.Q^T: 8 elements of head head0 + g per 32-element slice of the row,
// zero past the group's heads
template <int D, typename TQ>
__device__ __forceinline__ void decode_attn_load_q(uint4 (&qf)[D / 32], const TQ* q, const DecodeAttnItem& cta,
                                                   int num_heads, int g, int t) {
#pragma unroll
    for (int i = 0; i < D / 32; ++i)
        qf[i] = (g < cta.mq) ? ld_cg_u4(q + ((size_t)cta.bq * num_heads + cta.head0 + g) * D + i * 32 + t * 8)
                           : make_uint4(0, 0, 0, 0);
}

// element d of q head h of the group: the output itself when the launch has one split, else the split's partial for
// k_attn_combine (o already divided by l, with the split's max m and sum l)
template <typename T, int D>
__device__ __forceinline__ void decode_attn_store(const DecodeAttnItem& cta, int h, int d, float v, float m, float l,
                                                  int num_heads, int num_splits, T* out, float* part_o, float* part_m,
                                                  float* part_l) {
    const size_t vh = (size_t)cta.bq * num_heads + cta.head0 + h;
    if (num_splits == 1) {
        out[vh * D + d] = from_f32<T>(v);
    } else {
        part_o[(vh * num_splits + cta.split) * D + d] = v;
        if (d == 0) {
            part_m[vh * num_splits + cta.split] = m;
            part_l[vh * num_splits + cta.split] = l;
        }
    }
}

// k_decode_attn and k_decode_attn_kv8: sum the warps' P.V accumulators s_red [warp][head 8][D], divide by each head's
// sum and store
template <typename T, int D>
__device__ __forceinline__ void decode_attn_reduce_store(const DecodeAttnItem& cta, const float* s_red, const float* s_m,
                                                         const float* s_l, int num_heads, int num_splits, T* out,
                                                         float* part_o, float* part_m, float* part_l) {
    for (int e = threadIdx.x; e < cta.mq * D; e += kAttnThreads) {
        const int h = e / D, d = e % D;
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < kAttnWarps; ++k) v += s_red[(k * 8 + h) * D + d];
        decode_attn_store<T, D>(cta, h, d, v / s_l[h], s_m[h], s_l[h], num_heads, num_splits, out, part_o, part_m,
                                part_l);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Merge of key-split partials with the reference's LSE rule (attention_kernel.cu:881-923).
// grid (rows * num_heads), block D.  part_o ((vh * num_splits + split) * D + d) holds each split's output already
// divided by its own sum, part_m / part_l (vh * num_splits + split) its max and sum.
// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_attn_combine(const float* __restrict__ part_o, const float* __restrict__ part_m,
                               const float* __restrict__ part_l, T* __restrict__ out, int num_splits) {
    const int vh = blockIdx.x, D = blockDim.x, d = threadIdx.x;
    pdl_trigger();
    pdl_wait();
    const float* pm = part_m + (size_t)vh * num_splits;
    const float* pl = part_l + (size_t)vh * num_splits;
    float gm = -1e20f;
    for (int i = 0; i < num_splits; ++i) gm = fmaxf(gm, pm[i]);
    float gs = 0.f;
    for (int i = 0; i < num_splits; ++i) gs += pl[i] * expf(pm[i] - gm);
    float res = 0.f;
    for (int i = 0; i < num_splits; ++i) {
        const float w = pl[i] / gs * expf(pm[i] - gm);
        res += part_o[((size_t)vh * num_splits + i) * D + d] * w;
    }
    out[(size_t)vh * D + d] = from_f32<T>(res);
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------

// key splits of k_decode_attn and k_decode_attn_kv8: about two CTAs per SM, at least 256 keys per split, at most 64
// splits unless a split would exceed kAttnMaxRange keys
inline int attn_num_splits(int B, int len_q, int num_kv_heads, int m_query, int max_len_buf) {
    const int hgroups = (m_query + 7) / 8;
    const int base = B * len_q * num_kv_heads * hgroups;
    const int min_splits = cdiv(max_len_buf, kAttnMaxRange);
    const int want = cdiv(2 * device_sm_count(), base);
    const int max_useful = cdiv(max_len_buf, 256) > 0 ? cdiv(max_len_buf, 256) : 1;   // >= 256 keys per split
    int s = want < max_useful ? want : max_useful;
    if (s > kAttnMaxSplits) s = kAttnMaxSplits;
    if (s < min_splits) s = min_splits;
    if (s < 1) s = 1;
    return s;
}

// The split partials k_attn_combine reads, carved from the caller's workspace: o (vheads, splits, dv) fp32, then m and
// l (vheads, splits).  All null when the launch has one split and writes its output directly.
struct AttnParts {
    float* o;
    float* m;
    float* l;
};
inline size_t attn_parts_bytes(size_t vheads, int splits, int dv) {
    return vheads * splits * (dv + 2) * sizeof(float);
}
inline AttnParts attn_parts(void* ws, size_t vheads, int splits, int dv) {
    if (splits <= 1) return {nullptr, nullptr, nullptr};
    float* o = static_cast<float*>(ws);
    float* m = o + vheads * splits * dv;
    return {o, m, m + vheads * splits};
}

// k_attn_combine over the partials of a launch with `splits` key splits; nothing to do for one split
template <typename T>
inline cudaError_t launch_attn_combine(const AttnParts& p, size_t vheads, int dv, T* out, int splits,
                                       cudaStream_t stream, bool pdl) {
    if (splits <= 1) return cudaSuccess;
    return launch(k_attn_combine<T>, dim3((unsigned)vheads), dim3(dv), 0, stream, pdl, (const float*)p.o,
                  (const float*)p.m, (const float*)p.l, out, splits);
}

// Kernel's opt-in to `bytes` of dynamic shared memory (above the default 48 KiB), set once per device: the attribute
// belongs to the current device, and one process may drive several.
template <auto Kernel>
inline cudaError_t attn_smem_opt_in(int bytes) {
    static bool done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && done[dev]) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && dev >= 0 && dev < 64) done[dev] = true;
    return e;
}

}  // namespace zl
