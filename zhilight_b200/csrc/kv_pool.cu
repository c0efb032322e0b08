// KV row copies of the decode driver, one launch for every layer, K and V, and with an int8 cache the per-row fp32 scales
// with the codes:
//   - the prompt prefix cache: fixed-size token blocks between a task's rows and the model's device block pool
//     (zl_llama_kv_blocks_save / zl_llama_kv_blocks_load).  Stands in for PrefixCache::save_block / load_block (reference
//     src/generator/prefix_cache.hpp:48-58), which issue one dump_slice / load_slice per (block, K|V) for every layer;
//   - beam forks: row ranges from one task's rows into another's (zl_llama_kv_copy_rows);
//   - the KV arena: tasks moved and granted rows inside the row space, with their pointer tables rewritten
//     (k_kv_relocate; RagBufferContext::resize_task_buf, reference src/model/rag_buffer_context.h:119-133, reallocates
//     and copies a task's buffer per layer instead).
// A task's rows are reached through the live per-task pointer tables, so the copies follow the arena's moves.
#include "common.cuh"
#include "kv_pool.cuh"

namespace zl {
namespace {

constexpr int kCopyThreads = 256;
constexpr int kCopyVec = 4;                                   // loads in flight per thread

template <typename W>
constexpr int piece_bytes() { return kCopyThreads * kCopyVec * (int)sizeof(W); }   // bytes one CTA moves per step
constexpr int kPieceBytes = piece_bytes<uint4>();

// Piece `piece` of a range of `bytes` bytes, in words W: the first copy_bytes are loaded in full before they are stored,
// the rest is zero-filled.
template <typename W>
__device__ __forceinline__ void move_piece(const char* src, char* dst, int copy_bytes, int bytes, int piece) {
    const int step = kCopyThreads * (int)sizeof(W);
    const int off0 = piece * piece_bytes<W>() + threadIdx.x * (int)sizeof(W);
    W v[kCopyVec];
#pragma unroll
    for (int i = 0; i < kCopyVec; ++i) {
        const int off = off0 + i * step;
        if (off < copy_bytes) v[i] = *reinterpret_cast<const W*>(src + off);
    }
#pragma unroll
    for (int i = 0; i < kCopyVec; ++i) {
        const int off = off0 + i * step;
        if (off < copy_bytes)
            *reinterpret_cast<W*>(dst + off) = v[i];
        else if (off < bytes)
            *reinterpret_cast<W*>(dst + off) = W{};
    }
}

template <typename W>
__device__ __forceinline__ void copy_piece(const char* src, char* dst, int bytes, int piece) {
    move_piece<W>(src, dst, bytes, bytes, piece);
}

// The grid-stride loop of the three copy kernels over pieces of (item, layer, tensor, chunk): first the K / V pieces of
// every unit (ppk each), then the scale pieces (pps each).  f(scales, piece, item, layer, tensor).
template <typename F>
__device__ __forceinline__ void for_each_piece(int items, int layers, int ppk, int pps, F&& f) {
    const long long units = (long long)items * layers * 2;
    const long long kv_pieces = units * ppk, total = kv_pieces + units * pps;
    for (long long p = blockIdx.x; p < total; p += gridDim.x) {
        const bool sc = p >= kv_pieces;
        const long long q = sc ? p - kv_pieces : p;
        const int per = sc ? pps : ppk;
        const long long u = q / per;
        f(sc, (int)(q % per), (int)((u >> 1) / layers), (int)((u >> 1) % layers), (int)(u & 1));
    }
}

// Every K / V block (bt * row_bytes bytes each), then every scale block (bt * srow_bytes).
__global__ void __launch_bounds__(kCopyThreads, 8) k_kv_block_copy(KvBlockCopyArgs a) {
    const int blk = a.bt * a.row_bytes, sblk = a.bt * a.srow_bytes;
    for_each_piece(a.n, a.layers, (blk + kPieceBytes - 1) / kPieceBytes, (sblk + kPieceBytes - 1) / kPieceBytes,
                   [&](bool sc, int piece, int pair, int layer, int tensor) {
                       const int tb = a.pairs[pair], pb = a.pairs[a.n + pair];
                       const int bytes = sc ? sblk : blk;
                       char* task = static_cast<char*>(a.task_tabs[layer * 4 + (sc ? 2 : 0) + tensor][a.task]) +
                                    (size_t)tb * bytes;
                       char* pool = (sc ? a.pool_scales : a.pool) +
                                    ((size_t)(layer * 2 + tensor) * a.num_blocks + pb) * bytes;
                       const char* src = a.to_pool ? task : pool;
                       char* dst = a.to_pool ? pool : task;
                       copy_piece<uint4>(src, dst, bytes, piece);
                   });
}

// The K / V rows of every range in 16-byte words, then their scale rows in 4-byte words (a scale row of H_kv floats need
// not start on 16 bytes).  Every range gets the pieces of the longest one; the surplus pieces copy nothing.
__global__ void __launch_bounds__(kCopyThreads, 8) k_kv_row_copy(KvRowCopyArgs a) {
    for_each_piece(a.n, a.layers, (a.max_rows * a.row_bytes + kPieceBytes - 1) / kPieceBytes,
                   (a.max_rows * a.srow_bytes + piece_bytes<uint32_t>() - 1) / piece_bytes<uint32_t>(),
                   [&](bool sc, int piece, int range, int layer, int tensor) {
                       const int32_t* r4 = a.ranges + 4 * range;   // {src task, dst task, row0, row1}
                       const int rb = sc ? a.srow_bytes : a.row_bytes;
                       const int bytes = (r4[3] - r4[2]) * rb;
                       void* const* tab = a.task_tabs[layer * 4 + (sc ? 2 : 0) + tensor];
                       const char* src = static_cast<const char*>(tab[r4[0]]) + (size_t)r4[2] * rb;
                       char* dst = static_cast<char*>(tab[r4[1]]) + (size_t)r4[2] * rb;
                       if (sc)
                           copy_piece<uint32_t>(src, dst, bytes, piece);
                       else
                           copy_piece<uint4>(src, dst, bytes, piece);
                   });
}

// The moves' K / V rows in 16-byte words, then their scale rows in 4-byte words, each copied and then zero-filled past the
// copied rows; pieces as in k_kv_row_copy.  CTA 0 also rewrites the per-task tables: no kernel of this launch reads
// them, and every later kernel on the stream sees the new entries.  6 CTAs per SM: the zero fill and the table rewrite
// spill at the 32 registers of 8.
constexpr int kRelocateCtasPerSm = 6;
__global__ void __launch_bounds__(kCopyThreads, kRelocateCtasPerSm) k_kv_relocate(KvRelocateArgs a) {
    if (a.tabs && blockIdx.x == 0) {
        for (int i = threadIdx.x; i < a.layers * 4 * a.n_tasks; i += kCopyThreads) {
            const int lt = i / a.n_tasks, task = i % a.n_tasks;
            const int rb = (lt & 2) ? a.srow_bytes : a.row_bytes;
            if (rb) a.tabs[lt][task] = static_cast<char*>(a.bases[lt]) + (size_t)a.firsts[task] * rb;
        }
    }
    for_each_piece(a.n, a.layers, (a.max_rows * a.row_bytes + kPieceBytes - 1) / kPieceBytes,
                   (a.max_rows * a.srow_bytes + piece_bytes<uint32_t>() - 1) / piece_bytes<uint32_t>(),
                   [&](bool sc, int piece, int move, int layer, int tensor) {
                       const int32_t* m4 = a.moves + 4 * move;   // {src row, dst row, copy, zero}
                       const int rb = sc ? a.srow_bytes : a.row_bytes;
                       char* base = static_cast<char*>(a.bases[layer * 4 + (sc ? 2 : 0) + tensor]);
                       const char* src = base + (size_t)m4[0] * rb;
                       char* dst = base + (size_t)m4[1] * rb;
                       if (sc)
                           move_piece<uint32_t>(src, dst, m4[2] * rb, (m4[2] + m4[3]) * rb, piece);
                       else
                           move_piece<uint4>(src, dst, m4[2] * rb, (m4[2] + m4[3]) * rb, piece);
                   });
}

int copy_grid(long long pieces, int per_sm = 8) {
    // per_sm resident CTAs of 256 threads (8 fill an SM); more would only queue
    const long long cap = (long long)per_sm * device_sm_count();
    return (int)(pieces < 1 ? 1 : pieces < cap ? pieces : cap);
}

// pieces of n items of max_rows rows: K / V in 16-byte words, scales in 4-byte words
long long row_pieces(int n, int layers, int max_rows, int row_bytes, int srow_bytes) {
    return (long long)n * layers * 2 *
           (cdiv(max_rows * row_bytes, kPieceBytes) + cdiv(max_rows * srow_bytes, piece_bytes<uint32_t>()));
}

}  // namespace

bool kv_block_copy_aligned(int bt, int unit, int row_bytes, int srow_bytes) {
    // block offsets are multiples of bt rows; task bases multiples of unit rows
    for (int rb : {row_bytes, srow_bytes})
        if (((size_t)bt * rb) % 16 != 0 || ((size_t)unit * rb) % 16 != 0) return false;
    return true;
}

int kv_block_copy(const KvBlockCopyArgs& a, cudaStream_t stream) {
    ZL_CHECK_ARG(a.n > 0 && a.layers > 0 && a.pairs && a.task_tabs && a.pool);
    ZL_CHECK_ARG(!a.srow_bytes || a.pool_scales);
    const long long units = (long long)a.n * a.layers * 2;
    const long long pieces = units * (cdiv(a.bt * a.row_bytes, kPieceBytes) + cdiv(a.bt * a.srow_bytes, kPieceBytes));
    ZL_CHECK_CUDA(launch(k_kv_block_copy, dim3(copy_grid(pieces)), dim3(kCopyThreads), 0, stream, false, a));
    return ZL_OK;
}

int kv_row_copy(const KvRowCopyArgs& a, cudaStream_t stream) {
    ZL_CHECK_ARG(a.n > 0 && a.layers > 0 && a.max_rows > 0 && a.ranges && a.task_tabs);
    ZL_CHECK_ARG(a.row_bytes % 16 == 0 && a.srow_bytes % 4 == 0);
    const long long pieces = row_pieces(a.n, a.layers, a.max_rows, a.row_bytes, a.srow_bytes);
    ZL_CHECK_CUDA(launch(k_kv_row_copy, dim3(copy_grid(pieces)), dim3(kCopyThreads), 0, stream, false, a));
    return ZL_OK;
}

int kv_relocate(const KvRelocateArgs& a, cudaStream_t stream) {
    ZL_CHECK_ARG(a.n >= 0 && a.layers > 0 && a.bases && (a.n == 0 || (a.moves && a.max_rows > 0)));
    ZL_CHECK_ARG(a.n > 0 || a.tabs);
    ZL_CHECK_ARG(!a.tabs || (a.firsts && a.n_tasks > 0));
    ZL_CHECK_ARG(a.row_bytes % 16 == 0 && a.srow_bytes % 4 == 0);
    ZL_CHECK_ARG((long long)a.max_rows * a.row_bytes < (1LL << 31));   // byte offsets inside a move are int
    const long long pieces = row_pieces(a.n, a.layers, a.max_rows, a.row_bytes, a.srow_bytes);
    ZL_CHECK_CUDA(launch(k_kv_relocate, dim3(copy_grid(pieces, kRelocateCtasPerSm)), dim3(kCopyThreads), 0, stream, false, a));
    return ZL_OK;
}

}  // namespace zl

extern "C" int zl_kv_relocate(void* const* bases, int layers, const int32_t* moves, int n, int max_rows, int row_bytes,
                              int srow_bytes, zl_stream_t stream) {
    ZL_CHECK_ARG(n > 0);
    zl::KvRelocateArgs a{};
    a.bases = bases;
    a.moves = moves;
    a.n = n;
    a.layers = layers;
    a.max_rows = max_rows;
    a.row_bytes = row_bytes;
    a.srow_bytes = srow_bytes;
    return zl::kv_relocate(a, (cudaStream_t)stream);
}
