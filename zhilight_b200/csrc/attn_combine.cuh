// Merge of key-split attention partials with the reference's LSE rule (attention_kernel.cu:881-923), shared by the
// decode attention kernels and the variable-length attention kernel.
#pragma once
#include "common.cuh"

namespace zl {

// grid (rows * num_heads), block D.  part_o ((vh * num_splits + split) * D + d) holds each split's output already
// divided by its own sum, part_m / part_l (vh * num_splits + split) its max and sum.
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

}  // namespace zl
