// Block copies between a task's KV rows and the prompt-prefix block pool of the decode driver (kv_pool.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace zl {

// One launch moves n blocks of one task, every layer, K and V (and their fp32 scales with an int8 cache).
//   task side: block j = rows [j bt, (j + 1) bt) of the task's (max_seq, H_kv, d) buffer -- one contiguous range per
//              (layer, tensor); task_bases[4 l + t] is layer l's buffer of all tasks, t = 0 K, 1 V, 2 K scales, 3 V scales
//   pool side: pool [layer][K|V][pool block][bt][row_bytes], pool_scales [layer][K|V][pool block][bt][srow_bytes]
struct KvBlockCopyArgs {
    void* const* task_bases;   // device table, 4 per layer (scale entries unused without scales)
    char* pool;
    char* pool_scales;         // nullptr: no scales (srow_bytes == 0)
    const int32_t* pairs;      // device: n task blocks, then the n matching pool blocks
    int n, layers, num_blocks, bt;
    int task, task_rows;       // task_rows = max_seq
    int row_bytes, srow_bytes;
    int to_pool;               // 1: task -> pool (save), 0: pool -> task (load)
};

// every address the kernel forms is 16-byte aligned for these geometries
bool kv_block_copy_aligned(int bt, int task_rows, int row_bytes, int srow_bytes);
int kv_block_copy(const KvBlockCopyArgs& a, cudaStream_t stream);

// One launch copies n row ranges between tasks, every layer, K and V (and their fp32 scales with an int8 cache): range i
// = ranges[4 i ..] {src task, dst task, row0, row1} moves rows [row0, row1) of the src task's (max_seq, H_kv, d) buffers
// to the same rows of the dst task's.  No task may be both a source and a destination, and no destination may repeat.
struct KvRowCopyArgs {
    void* const* task_bases;   // device table, 4 per layer as in KvBlockCopyArgs
    const int32_t* ranges;     // device (n, 4)
    int n, layers, task_rows, max_rows;   // max_rows: the longest range
    int row_bytes, srow_bytes;            // row_bytes % 16 == 0; srow_bytes 0 (no scales) or a multiple of 4
};
int kv_row_copy(const KvRowCopyArgs& a, cudaStream_t stream);

}  // namespace zl
