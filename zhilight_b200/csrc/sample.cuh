// The sampler (sample.cu) as the decode driver runs it.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/zhilight_b200.h"

namespace zl {

// Per-task token automata on the device (zl_llama_set_constraint).  Task t in state s >= 0 (state[t], or t itself when
// state is NULL) keeps only the tokens of mask row (t * states + s): words u32 per row, bit j of word i = token 32 i + j.
// With next non-NULL the pick x of a recorded row moves the task to next[t * max_edges + e] for the edge e in
// [row_ptr[t * (states + 1) + s], row_ptr[t * (states + 1) + s + 1]) whose edge_tok is x (sorted per state), else to
// dflt[t * states + s]; state[t] < 0: the task is unconstrained.  next NULL: the state is only read.
// zl_sample_masked uses this as a plain per-task mask table: states = 0 and state = its mask_row, so task t reads mask
// row mask_row[t] (t when NULL), and next = NULL, so nothing is written through state.
struct SampleAutomata {
    const uint32_t* mask = nullptr;
    int32_t* state = nullptr;
    int words = 0, states = 0, max_edges = 0;
    const int32_t *row_ptr = nullptr, *edge_tok = nullptr, *next = nullptr, *dflt = nullptr;
};

// zl_sample_processed, plus frozen (tasks) or NULL: a row whose task has frozen[task] != 0 is picked as usual but its
// pick is recorded in neither the history bitmap nor the sequence, and moves no automaton (zl_llama_generate's finished
// tasks); au NULL or the tasks' automata (zl_sample_masked's contract for the mask)
int sample_processed_launch(const float* logits, int T, int V, const zl_sample_params_t* params, const int32_t* row_task,
                            const int32_t* counter, uint32_t* history, int history_words, const float* ngram_penalty,
                            int32_t* seq, int32_t* seq_len, int seq_stride, const int32_t* bias_tokens,
                            const float* bias_values, const int32_t* bias_count, int bias_stride, const int32_t* frozen,
                            const SampleAutomata* au, int32_t* out, void* ws, size_t ws_bytes, int pdl, cudaStream_t stream);

}  // namespace zl
