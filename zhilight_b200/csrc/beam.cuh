// Beam-search selection (beam.cu) as the decode driver runs it: host checks, then the launches over device groups.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace zl {

// zl_beam_topk's argument checks on a HOST groups array
int beam_topk_check(int R, int V, const int32_t* groups_host, int G, int K);
// zl_beam_topk's two launches with the groups already on the device; ws: zl_beam_topk_workspace_bytes(R, V, K)
int beam_topk_launch(const float* logits, int R, int V, const float* cum, const int32_t* groups, int G, int K,
                     int32_t* parent, int32_t* token, float* score, void* ws, int pdl, cudaStream_t stream);

}  // namespace zl
