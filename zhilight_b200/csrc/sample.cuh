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

// The processors' device arguments (zl_sample_processed); all NULL for zl_sample.
struct SampleProc {
    const float* ngram;       // (tasks) or NULL: no n-gram rule
    int32_t* seq;             // (tasks, seq_stride) generated tokens, oldest first, or NULL
    int32_t* seq_len;         // (tasks)
    int seq_stride;
    const int32_t* bias_tok;  // (tasks, bias_stride) or NULL
    const float* bias_val;
    const int32_t* bias_cnt;  // (tasks)
    int bias_stride;
    int2* table;              // k_ngram_levels' output: per row, table_stride {token, level} slots
    int table_stride;
    const int32_t* frozen;    // (tasks) or NULL: a row whose task has frozen[task] != 0 records its pick nowhere
    SampleAutomata au;        // au.mask NULL: no row is masked
};

// hash table slots for n distinct tokens at most: a power of two >= 2n, so an insert always finds a free slot
__host__ __device__ inline int ngram_table_size(int n) {
    int h = 2;
    while (h < 2 * n) h <<= 1;
    return h;
}

// zl_sample over the processors of pr: zl_sample_processed's contract, plus pr.frozen (zl_llama_generate's finished
// tasks: a frozen task's pick is recorded in neither the history bitmap nor the sequence, and moves no automaton) and
// pr.au (zl_sample_masked's contract for the mask).  pr.table must hold T rows.
int sample_launch(const float* logits, int T, int V, const zl_sample_params_t* params, const int32_t* row_task,
                  const int32_t* counter, uint32_t* history, int history_words, const SampleProc& pr, int32_t* out,
                  int pdl, cudaStream_t stream);

}  // namespace zl
