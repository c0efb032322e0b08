// Prompt prefix cache of the decode driver: copies of fixed-size token blocks of KV rows between a task's buffers and the
// model's device block pool (zl_llama_kv_blocks_save / zl_llama_kv_blocks_load).  Stands in for PrefixCache::save_block /
// load_block (reference src/generator/prefix_cache.hpp:48-58), which issue one dump_slice / load_slice per (block, K|V) for
// every layer; here one launch moves every layer, K and V, and with an int8 cache the per-row fp32 scales with the codes.
#include "common.cuh"
#include "kv_pool.cuh"

namespace zl {
namespace {

constexpr int kCopyThreads = 256;
constexpr int kCopyVec = 4;                                   // 16-byte loads in flight per thread
constexpr int kPieceBytes = kCopyThreads * kCopyVec * 16;     // bytes one CTA moves per grid-stride step

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
        const int off0 = piece * kPieceBytes + threadIdx.x * 16;
        uint4 v[kCopyVec];
#pragma unroll
        for (int i = 0; i < kCopyVec; ++i) {
            const int off = off0 + i * kCopyThreads * 16;
            if (off < bytes) v[i] = *reinterpret_cast<const uint4*>(src + off);
        }
#pragma unroll
        for (int i = 0; i < kCopyVec; ++i) {
            const int off = off0 + i * kCopyThreads * 16;
            if (off < bytes) *reinterpret_cast<uint4*>(dst + off) = v[i];
        }
    }
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
    // 8 resident CTAs of 256 threads fill an SM; more would only queue
    const long long cap = 8LL * device_sm_count();
    const int grid = (int)(pieces < cap ? pieces : cap);
    ZL_CHECK_CUDA(launch(k_kv_block_copy, dim3(grid), dim3(kCopyThreads), 0, stream, false, a));
    return ZL_OK;
}

}  // namespace zl
