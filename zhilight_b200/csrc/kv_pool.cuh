// KV row copies of the decode driver (kv_pool.cu): between a task's rows and the prompt-prefix block pool, between
// tasks, and the relocation of tasks inside the KV row space.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace zl {

// One launch moves n blocks of one task, every layer, K and V (and their fp32 scales with an int8 cache).
//   task side: block j = rows [j bt, (j + 1) bt) of the task's rows -- one contiguous range per (layer, tensor) from the
//              live per-task pointer table task_tabs[4 l + t][task]; t = 0 K, 1 V, 2 K scales, 3 V scales
//   pool side: pool [layer][K|V][pool block][bt][row_bytes], pool_scales [layer][K|V][pool block][bt][srow_bytes]
struct KvBlockCopyArgs {
    void* const* const* task_tabs;   // device, 4 per layer: the layer's per-task tables (scale entries unused without scales)
    char* pool;
    char* pool_scales;         // nullptr: no scales (srow_bytes == 0)
    const int32_t* pairs;      // device: n task blocks, then the n matching pool blocks
    int n, layers, num_blocks, bt;
    int task;
    int row_bytes, srow_bytes;
    int to_pool;               // 1: task -> pool (save), 0: pool -> task (load)
};

// every address the kernel forms is 16-byte aligned for these geometries (task bases are multiples of `unit` rows)
bool kv_block_copy_aligned(int bt, int unit, int row_bytes, int srow_bytes);
int kv_block_copy(const KvBlockCopyArgs& a, cudaStream_t stream);

// One launch copies n row ranges between tasks, every layer, K and V (and their fp32 scales with an int8 cache): range i
// = ranges[4 i ..] {src task, dst task, row0, row1} moves rows [row0, row1) of the src task to the same rows of the dst
// task, both reached through the live per-task tables.  No task may be both a source and a destination, and no
// destination may repeat.
struct KvRowCopyArgs {
    void* const* const* task_tabs;   // device, 4 per layer as in KvBlockCopyArgs
    const int32_t* ranges;     // device (n, 4)
    int n, layers, max_rows;   // max_rows: the longest range
    int row_bytes, srow_bytes; // row_bytes % 16 == 0; srow_bytes 0 (no scales) or a multiple of 4
};
int kv_row_copy(const KvRowCopyArgs& a, cudaStream_t stream);

// One launch (k_kv_relocate) applies n moves {src row, dst row, rows to copy, rows to zero} of the row space (KvMove),
// every layer, K and V (and their scales): rows [src, src + copy) to [dst, dst + copy), then rows [dst + copy, dst + copy +
// zero) zero-filled.  No move may overlap another's source or destination.  With tabs, the launch also rewrites every
// per-task table entry tabs[4 l + t][task] = bases[4 l + t] + firsts[task] * (row or scale-row bytes), task < n_tasks:
// the kernels that run after it reach the tasks' new rows.
struct KvRelocateArgs {
    void* const* bases;        // device, 4 per layer: the layer's row space of K, V, K scales, V scales
    const int32_t* moves;      // device (n, 4); n may be 0 with tabs
    int n, layers, max_rows;   // max_rows: the largest copy + zero
    int row_bytes, srow_bytes; // row_bytes % 16 == 0; srow_bytes 0 (no scales) or a multiple of 4
    void** const* tabs;        // device, 4 per layer, or nullptr
    const int32_t* firsts;     // device (n_tasks)
    int n_tasks;
};
int kv_relocate(const KvRelocateArgs& a, cudaStream_t stream);

}  // namespace zl
