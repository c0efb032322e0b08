// The sampler (sample.cu) as the decode driver runs it.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/zhilight_b200.h"

namespace zl {

// zl_sample_processed, plus frozen (tasks) or NULL: a row whose task has frozen[task] != 0 is picked as usual but its
// pick is recorded in neither the history bitmap nor the sequence (zl_llama_generate's finished tasks)
int sample_processed_launch(const float* logits, int T, int V, const zl_sample_params_t* params, const int32_t* row_task,
                            const int32_t* counter, uint32_t* history, int history_words, const float* ngram_penalty,
                            int32_t* seq, int32_t* seq_len, int seq_stride, const int32_t* bias_tokens,
                            const float* bias_values, const int32_t* bias_count, int bias_stride, const int32_t* frozen,
                            int32_t* out, void* ws, size_t ws_bytes, int pdl, cudaStream_t stream);

}  // namespace zl
