// Vocabulary all-gather over NVLink peer memory: every rank's (T, vshard) fp32 lm_head shard lands in columns
// [rank * vshard, (rank + 1) * vshard) of a (T, V) row-major fp32 buffer on every rank, so that the sampler and the
// beam selection read full-vocabulary rows under tensor parallelism.  The reference all-gathers the logit shards with
// NCCL before its pick (src/nn/embedding/embedding.cu:353-390); here one kernel pushes the shard straight into the peers'
// buffers, mapped with CUDA IPC, and the picks read the buffer in place.
//
// A separate exchange object from zl_comm: its inboxes scale with the all-reduce message and hold two parities per
// source, which a (max_rows, V) fp32 payload would multiply several times over.
//
// Overwrite safety with ONE buffer per rank: a peer's gather of step s + 1 must not land while this rank still reads the
// rows of step s.  Every forward of a tensor-parallel decoder runs at least one all-reduce before its lm_head, and that
// exchange completes on a peer only after this rank has published its part of it.  This rank publishes only after its
// pick of step s has finished: every step starts with a launch without programmatic dependency (k_lens_from_pos,
// k_prefill_setup), so everything of step s + 1 runs after the pick of step s in stream order.  Hence the peer's next
// gather, which follows its all-reduces in stream order, starts after this rank's pick of step s has finished.  A user
// of the bare gather (no forward between two gathers) must order its reads of the buffer the same way.
#include "common.cuh"
#include "comm_dev.cuh"

#include <cstring>

namespace zl {

constexpr int kVgThreads = 256;
constexpr int kVgUnroll = 4;   // 16-byte vectors each thread loads before it stores them

struct VocabGatherDev {                  // a kernel argument: the mapping is fixed once the peers are opened
    float* buf[kCommMaxRanks];           // buf[r] = rank r's (max_rows, V) buffer as mapped here
    size_t flags_off;                    // float offset of the flags [ws sources][kCommMaxCtas] (uint64, monotonic)
    unsigned long long* epoch;           // local: completed gathers
    unsigned int* done;                  // local: CTAs finished in the current gather
    int rank, ws, V, vshard;
};

__global__ void __launch_bounds__(kVgThreads)
k_vocab_gather(const __grid_constant__ VocabGatherDev g, const float* __restrict__ shard, int rows, int ld) {
    __shared__ unsigned long long s_epoch;
    pdl_trigger();
    pdl_wait();
    if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile unsigned long long*>(g.epoch);
    __syncthreads();
    const unsigned long long e = s_epoch;
    const int q = g.vshard / 4;   // 16-byte vectors per shard row
    const int n = rows * q;
    const int i0 = (int)((long long)n * blockIdx.x / gridDim.x), i1 = (int)((long long)n * (blockIdx.x + 1) / gridDim.x);
    const size_t col0 = (size_t)g.rank * g.vshard;

    // ---- push this CTA's chunk into every rank's buffer, this one's included ----
    for (int base = i0 + threadIdx.x; base < i1; base += kVgThreads * kVgUnroll) {
        uint4 v[kVgUnroll];
        size_t off[kVgUnroll];
#pragma unroll
        for (int k = 0; k < kVgUnroll; ++k) {
            const int i = base + k * kVgThreads;
            if (i < i1) {
                const int row = i / q, c = i - row * q;
                v[k] = ld_cg_u4(shard + (size_t)row * ld + 4 * c);
                off[k] = (size_t)row * g.V + col0 + 4 * c;
            }
        }
        for (int r = 0; r < g.ws; ++r) {
            float* dst = g.buf[r];
#pragma unroll
            for (int k = 0; k < kVgUnroll; ++k)
                if (base + k * kVgThreads < i1) *reinterpret_cast<uint4*>(dst + off[k]) = v[k];
        }
    }
    __threadfence_system();
    __syncthreads();
    // ---- publish the chunk, then wait for the same chunk of every peer ----
    if (threadIdx.x < g.ws && (int)threadIdx.x != g.rank) {
        unsigned long long* peer_flags = reinterpret_cast<unsigned long long*>(g.buf[threadIdx.x] + g.flags_off);
        st_release_sys(peer_flags + (size_t)g.rank * kCommMaxCtas + blockIdx.x, e + 1);
        const unsigned long long* mine =
            reinterpret_cast<const unsigned long long*>(g.buf[g.rank] + g.flags_off) + (size_t)threadIdx.x * kCommMaxCtas + blockIdx.x;
        while (ld_acquire_sys(mine) < e + 1) {
        }
    }
    // ---- last CTA out advances the epoch ----
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(g.done, 1u) == gridDim.x - 1) {
            *g.done = 0;
            __threadfence();
            *reinterpret_cast<volatile unsigned long long*>(g.epoch) = e + 1;
        }
    }
}

}  // namespace zl

using namespace zl;

struct zl_vocab_gather {
    int rank = 0, ws = 1, max_rows = 0, V = 0;
    float* local = nullptr;                 // this rank's buffer: (max_rows, V) fp32, then the flags
    float* peers[kCommMaxRanks] = {};       // mapped peer buffers (peers[rank] == local)
    unsigned long long* epoch = nullptr;
    unsigned int* done = nullptr;
    bool opened = false;
};

namespace {

size_t flags_off(const zl_vocab_gather* g) { return ((size_t)g->max_rows * g->V + 31) / 32 * 32; }   // 128-byte aligned

}  // namespace

extern "C" int zl_vocab_gather_create(int rank, int world_size, int max_rows, int vocab, zl_vocab_gather_t** out) {
    ZL_CHECK_ARG(out && world_size >= 1 && world_size <= kCommMaxRanks && rank >= 0 && rank < world_size);
    ZL_CHECK_ARG(max_rows >= 1 && vocab >= 1 && vocab % world_size == 0);
    ZL_CHECK_SUPPORTED((vocab / world_size) % 4 == 0);   // 16-byte vectors of the shard rows
    ZL_CHECK_ARG((long long)max_rows * vocab < (1LL << 31));
    zl_vocab_gather* g = new zl_vocab_gather();
    g->rank = rank;
    g->ws = world_size;
    g->max_rows = max_rows;
    g->V = vocab;
    const size_t bytes = (flags_off(g) + (size_t)2 * world_size * kCommMaxCtas) * sizeof(float);
    auto fail = [&](cudaError_t e) {
        cudaFree(g->local);
        cudaFree(g->epoch);
        cudaFree(g->done);
        delete g;
        zl_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e));
        return ZL_ERR_CUDA;
    };
    cudaError_t e = cudaMalloc((void**)&g->local, bytes);
    if (e == cudaSuccess) e = cudaMemset(g->local, 0, bytes);
    if (e == cudaSuccess) e = cudaMalloc((void**)&g->epoch, 8);
    if (e == cudaSuccess) e = cudaMemset(g->epoch, 0, 8);
    if (e == cudaSuccess) e = cudaMalloc((void**)&g->done, 4);
    if (e == cudaSuccess) e = cudaMemset(g->done, 0, 4);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return fail(e);
    g->peers[rank] = g->local;
    g->opened = world_size == 1;
    *out = g;
    return ZL_OK;
}

extern "C" int zl_vocab_gather_get_ipc_handle(zl_vocab_gather_t* g, void* handle_out) {
    ZL_CHECK_ARG(g && handle_out);
    cudaIpcMemHandle_t h;
    ZL_CHECK_CUDA(cudaIpcGetMemHandle(&h, g->local));
    memcpy(handle_out, &h, sizeof(h));
    return ZL_OK;
}

// handles_all: world_size consecutive cudaIpcMemHandle_t, index = rank (the own entry is ignored)
extern "C" int zl_vocab_gather_open_peers(zl_vocab_gather_t* g, const void* handles_all) {
    ZL_CHECK_ARG(g && handles_all);
    if (g->opened) return ZL_OK;
    const cudaIpcMemHandle_t* hs = static_cast<const cudaIpcMemHandle_t*>(handles_all);
    for (int r = 0; r < g->ws; ++r) {
        if (r == g->rank || g->peers[r]) continue;
        void* p = nullptr;
        ZL_CHECK_CUDA(cudaIpcOpenMemHandle(&p, hs[r], cudaIpcMemLazyEnablePeerAccess));
        g->peers[r] = static_cast<float*>(p);
    }
    g->opened = true;
    return ZL_OK;
}

extern "C" int zl_vocab_gather_info(zl_vocab_gather_t* g, int* rank, int* world_size, int* max_rows, int* vocab) {
    ZL_CHECK_ARG(g && rank && world_size && max_rows && vocab);
    *rank = g->rank;
    *world_size = g->ws;
    *max_rows = g->max_rows;
    *vocab = g->V;
    return ZL_OK;
}

extern "C" float* zl_vocab_gather_buffer(zl_vocab_gather_t* g) { return g ? g->local : nullptr; }

extern "C" int zl_vocab_allgather(zl_vocab_gather_t* g, const float* shard, int rows, int ld, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(g && shard && reinterpret_cast<uintptr_t>(shard) % 16 == 0);
    const int vshard = g->V / g->ws;
    ZL_CHECK_ARG(rows >= 1 && rows <= g->max_rows && ld >= vshard && ld % 4 == 0);
    if (!g->opened) {
        zl_set_last_error(__FILE__, __LINE__, "zl_vocab_allgather: peers not opened");
        return ZL_ERR_STATE;
    }
    VocabGatherDev d = {};
    for (int r = 0; r < g->ws; ++r) d.buf[r] = g->peers[r];
    d.flags_off = flags_off(g);
    d.epoch = g->epoch;
    d.done = g->done;
    d.rank = g->rank;
    d.ws = g->ws;
    d.V = g->V;
    d.vshard = vshard;
    // about one 16-byte vector per thread at decode sizes, and every CTA resident (the CTAs of all ranks wait for each other)
    const int n = rows * (vshard / 4);
    int ctas = cdiv(n, kVgThreads);
    if (ctas > kCommMaxCtas) ctas = kCommMaxCtas;
    ZL_CHECK_CUDA(launch(k_vocab_gather, dim3(ctas), dim3(kVgThreads), 0, stream, pdl != 0, d, shard, rows, ld));
    return ZL_OK;
}

extern "C" void zl_vocab_gather_destroy(zl_vocab_gather_t* g) {
    if (!g) return;
    cudaDeviceSynchronize();
    for (int r = 0; r < g->ws; ++r)
        if (r != g->rank && g->peers[r]) cudaIpcCloseMemHandle(g->peers[r]);
    cudaFree(g->local);
    cudaFree(g->epoch);
    cudaFree(g->done);
    delete g;
}
