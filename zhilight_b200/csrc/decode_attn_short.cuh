// Pieces shared by the decode attention kernels (decode_attn.cu, decode_attn_warp.cuh, decode_attn_kv8.cu, varlen_attn.cu):
// the per-type tensor-core MMA, key-range rounding, and the key range of one latency-regime CTA.
#pragma once
#include "common.cuh"

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

// keys per split in the latency regime (few CTAs of work), where zl_decode_attention runs the warp kernel
constexpr int kShortRange = 256;

}  // namespace zl
