// KV row copies of the decode driver, one launch for every layer, K and V, and with an int8 cache the per-row fp32 scales
// with the codes:
//   - the prompt prefix cache: fixed-size token blocks between a task's buffers and the model's device block pool
//     (zl_llama_kv_blocks_save / zl_llama_kv_blocks_load).  Stands in for PrefixCache::save_block / load_block (reference
//     src/generator/prefix_cache.hpp:48-58), which issue one dump_slice / load_slice per (block, K|V) for every layer;
//   - beam forks: row ranges from one task's buffers into another's (zl_llama_kv_copy_rows).
#include "common.cuh"
#include "kv_pool.cuh"

namespace zl {
namespace {

constexpr int kCopyThreads = 256;
constexpr int kCopyVec = 4;                                   // loads in flight per thread

template <typename W>
constexpr int piece_bytes() { return kCopyThreads * kCopyVec * (int)sizeof(W); }   // bytes one CTA moves per step
constexpr int kPieceBytes = piece_bytes<uint4>();

// Piece `piece` of a contiguous range of `bytes` bytes, in words W: loaded in full before it is stored.
template <typename W>
__device__ __forceinline__ void copy_piece(const char* src, char* dst, int bytes, int piece) {
    const int step = kCopyThreads * (int)sizeof(W);
    const int off0 = piece * piece_bytes<W>() + threadIdx.x * (int)sizeof(W);
    W v[kCopyVec];
#pragma unroll
    for (int i = 0; i < kCopyVec; ++i) {
        const int off = off0 + i * step;
        if (off < bytes) v[i] = *reinterpret_cast<const W*>(src + off);
    }
#pragma unroll
    for (int i = 0; i < kCopyVec; ++i) {
        const int off = off0 + i * step;
        if (off < bytes) *reinterpret_cast<W*>(dst + off) = v[i];
    }
}

// Grid-stride over pieces of (pair, layer, tensor, chunk): first every K / V block (bt * row_bytes bytes each), then every
// scale block (bt * srow_bytes).  A piece is kPieceBytes of one block, loaded in full before it is stored.
__global__ void __launch_bounds__(kCopyThreads, 8) k_kv_block_copy(KvBlockCopyArgs a) {
    const int blk = a.bt * a.row_bytes, sblk = a.bt * a.srow_bytes;
    const int ppk = (blk + kPieceBytes - 1) / kPieceBytes;
    const int pps = (sblk + kPieceBytes - 1) / kPieceBytes;
    const long long units = (long long)a.n * a.layers * 2;
    const long long kv_pieces = units * ppk, total = kv_pieces + units * pps;
    for (long long p = blockIdx.x; p < total; p += gridDim.x) {
        const bool sc = p >= kv_pieces;
        const long long q = sc ? p - kv_pieces : p;
        const int per = sc ? pps : ppk;
        const int piece = (int)(q % per);
        const long long u = q / per;
        const int tensor = (int)(u & 1);
        const int layer = (int)((u >> 1) % a.layers);
        const int pair = (int)((u >> 1) / a.layers);
        const int tb = a.pairs[pair], pb = a.pairs[a.n + pair];
        const int bytes = sc ? sblk : blk, rb = sc ? a.srow_bytes : a.row_bytes;
        char* task = static_cast<char*>(a.task_bases[layer * 4 + (sc ? 2 : 0) + tensor]) +
                     ((size_t)a.task * a.task_rows + (size_t)tb * a.bt) * rb;
        char* pool = (sc ? a.pool_scales : a.pool) + ((size_t)(layer * 2 + tensor) * a.num_blocks + pb) * bytes;
        const char* src = a.to_pool ? task : pool;
        char* dst = a.to_pool ? pool : task;
        copy_piece<uint4>(src, dst, bytes, piece);
    }
}

// Grid-stride over pieces of (range, layer, tensor, chunk): first the K / V rows of every range in 16-byte words, then
// their scale rows in 4-byte words (a scale row of H_kv floats need not start on 16 bytes).  Every range gets the pieces
// of the longest one; the surplus pieces copy nothing.
__global__ void __launch_bounds__(kCopyThreads, 8) k_kv_row_copy(KvRowCopyArgs a) {
    const int ppk = (a.max_rows * a.row_bytes + kPieceBytes - 1) / kPieceBytes;
    const int pps = (a.max_rows * a.srow_bytes + piece_bytes<uint32_t>() - 1) / piece_bytes<uint32_t>();
    const long long units = (long long)a.n * a.layers * 2;
    const long long kv_pieces = units * ppk, total = kv_pieces + units * pps;
    for (long long p = blockIdx.x; p < total; p += gridDim.x) {
        const bool sc = p >= kv_pieces;
        const long long q = sc ? p - kv_pieces : p;
        const int per = sc ? pps : ppk;
        const int piece = (int)(q % per);
        const long long u = q / per;
        const int tensor = (int)(u & 1);
        const int layer = (int)((u >> 1) % a.layers);
        const int range = (int)((u >> 1) / a.layers);
        const int32_t* r4 = a.ranges + 4 * range;   // {src task, dst task, row0, row1}
        const int rb = sc ? a.srow_bytes : a.row_bytes;
        const int bytes = (r4[3] - r4[2]) * rb;
        const char* base = static_cast<const char*>(a.task_bases[layer * 4 + (sc ? 2 : 0) + tensor]);
        const char* src = base + ((size_t)r4[0] * a.task_rows + r4[2]) * rb;
        char* dst = const_cast<char*>(base) + ((size_t)r4[1] * a.task_rows + r4[2]) * rb;
        if (sc)
            copy_piece<uint32_t>(src, dst, bytes, piece);
        else
            copy_piece<uint4>(src, dst, bytes, piece);
    }
}

int copy_grid(long long pieces) {
    // 8 resident CTAs of 256 threads fill an SM; more would only queue
    const long long cap = 8LL * device_sm_count();
    return (int)(pieces < cap ? pieces : cap);
}

}  // namespace

bool kv_block_copy_aligned(int bt, int task_rows, int row_bytes, int srow_bytes) {
    // block offsets are multiples of bt rows; task offsets multiples of task_rows rows
    for (int rb : {row_bytes, srow_bytes})
        if (((size_t)bt * rb) % 16 != 0 || ((size_t)task_rows * rb) % 16 != 0) return false;
    return true;
}

int kv_block_copy(const KvBlockCopyArgs& a, cudaStream_t stream) {
    ZL_CHECK_ARG(a.n > 0 && a.layers > 0 && a.pairs && a.task_bases && a.pool);
    ZL_CHECK_ARG(!a.srow_bytes || a.pool_scales);
    const long long units = (long long)a.n * a.layers * 2;
    const long long pieces = units * (cdiv(a.bt * a.row_bytes, kPieceBytes) + cdiv(a.bt * a.srow_bytes, kPieceBytes));
    ZL_CHECK_CUDA(launch(k_kv_block_copy, dim3(copy_grid(pieces)), dim3(kCopyThreads), 0, stream, false, a));
    return ZL_OK;
}

int kv_row_copy(const KvRowCopyArgs& a, cudaStream_t stream) {
    ZL_CHECK_ARG(a.n > 0 && a.layers > 0 && a.max_rows > 0 && a.ranges && a.task_bases);
    ZL_CHECK_ARG(a.row_bytes % 16 == 0 && a.srow_bytes % 4 == 0);
    const long long units = (long long)a.n * a.layers * 2;
    const long long pieces = units * (cdiv(a.max_rows * a.row_bytes, kPieceBytes) +
                                      cdiv(a.max_rows * a.srow_bytes, piece_bytes<uint32_t>()));
    ZL_CHECK_CUDA(launch(k_kv_row_copy, dim3(copy_grid(pieces)), dim3(kCopyThreads), 0, stream, false, a));
    return ZL_OK;
}

}  // namespace zl
