// Beam-search selection on the GPU: the K best (hypothesis, token) continuations of every group of rows, scored by the
// cumulative log-probability cum[r] + log_softmax(logits[r])[v], without materialising the (R, V) log-probabilities.
//
// Stands in for beam_utility::log_softmax_bias (reference src/generator/beam_util.cu:20-130: x - max - log(1e-20 + sum
// exp(x - max)) + bias per row) followed by topk_all.get_top_k over the flattened (beam x vocab) scores of each task
// (src/generator/batch_generator.cpp:1770-1778).
//
// The log-softmax is a per-row shift, so a group's top K lies in the union of its live rows' own top K, and a row's top K
// in the union of its chunks' top K.  Two launches:
//   1. k_beam_chunk, one CTA per (row chunk, row): the chunk's online (max, sum exp(x - max)) and its top K by
//      (logit descending, index ascending).  Dead rows (cum == -inf) return at once: their logits are never read.
//   2. k_beam_group, one CTA per group: the rows' log-sum-exp from the chunk statistics, the chunk lists shifted to scores,
//      and the group's top K by (score descending, flat index (r - row0) * V + v ascending).
// A running top K lives in one warp, lane j holding the j-th best entry; 32 candidates are tested against lane K-1 with
// one ballot, so most elements cost a compare.  One or two that pass are inserted with a shuffle, more are bitonic-sorted
// across the lanes and merged in, and the warps of a CTA merge their lists pairwise the same way.
#include "common.cuh"
#include "beam.cuh"

#include <climits>
#include <cstring>

namespace zl {
namespace {

constexpr int kBeamMaxK = 32;
constexpr int kBeamMaxWidth = 16;
constexpr int kBeamMaxVocab = 262144;   // flat indices (width * V) stay below 2^31
constexpr int kChunkThreads = 256;
constexpr int kGroupThreads = 512;
constexpr int kMaxChunks = 128;
constexpr int kMinChunk = 2048;         // elements a chunk CTA reads at least
constexpr int kTargetCtas = 1056;       // 8 resident chunk CTAs on each of 132 SMs
constexpr unsigned kFull = 0xffffffffu;

struct BeamCand {
    float v;
    int i;
};

__device__ __forceinline__ bool better(float av, int ai, float bv, int bi) { return av > bv || (av == bv && ai < bi); }

// A warp's running top K, sorted over all 32 lanes: lane j holds the j-th best (value, index); lanes >= K hold entries
// that no longer count.  thr is lane K-1's entry, the bar a candidate must clear.
struct WarpTopK {
    float v, tv;
    int i, ti;
    int K;

    __device__ void init(int k) {
        K = k;
        v = tv = -INFINITY;
        i = ti = INT_MAX;
    }
    // keeps the better of the entry of this lane and of lane ^ j: the lower lane the better one when `desc`
    __device__ static void exchange(float& v, int& i, int j, bool desc) {
        const float ov = __shfl_xor_sync(kFull, v, j);
        const int oi = __shfl_xor_sync(kFull, i, j);
        const bool lower = ((threadIdx.x & 31) & j) == 0;
        if (lower == desc ? better(ov, oi, v, i) : better(v, i, ov, oi)) {
            v = ov;
            i = oi;
        }
    }
    // merges a list sorted over the lanes (best first) into this one: the better of this lane's entry and the other
    // list's mirror entry form a bitonic sequence holding the best 32 of both, which 5 exchanges sort
    __device__ void merge_sorted(float cv, int ci) {
        const int lane = threadIdx.x & 31;
        const float rv = __shfl_sync(kFull, cv, 31 - lane);
        const int ri = __shfl_sync(kFull, ci, 31 - lane);
        if (better(rv, ri, v, i)) {
            v = rv;
            i = ri;
        }
#pragma unroll
        for (int j = 16; j > 0; j >>= 1) exchange(v, i, j, true);
        tv = __shfl_sync(kFull, v, K - 1);
        ti = __shfl_sync(kFull, i, K - 1);
    }
    // every lane offers one candidate (ok = false: none); warp-uniform call.  One or two that clear the bar are inserted
    // one by one; more are bitonic-sorted across the lanes and merged in.
    __device__ void offer(float cv, int ci, bool ok) {
        unsigned m = __ballot_sync(kFull, ok && better(cv, ci, tv, ti));
        if (__popc(m) > 2) {
            const int lane = threadIdx.x & 31;
            if (!((m >> lane) & 1)) {
                cv = -INFINITY;
                ci = INT_MAX;
            }
#pragma unroll
            for (int k = 2; k <= 32; k <<= 1)
#pragma unroll
                for (int j = k >> 1; j > 0; j >>= 1) exchange(cv, ci, j, ((threadIdx.x & 31) & k) == 0);
            merge_sorted(cv, ci);
            return;
        }
        const int lane = threadIdx.x & 31;
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const float xv = __shfl_sync(kFull, cv, src);
            const int xi = __shfl_sync(kFull, ci, src);
            if (!better(xv, xi, tv, ti)) continue;   // outranked by a candidate inserted in this loop
            const int pos = __popc(__ballot_sync(kFull, better(v, i, xv, xi)));
            const float uv = __shfl_up_sync(kFull, v, 1);
            const int ui = __shfl_up_sync(kFull, i, 1);
            if (lane > pos) {
                v = uv;
                i = ui;
            } else if (lane == pos) {
                v = xv;
                i = xi;
            }
            tv = __shfl_sync(kFull, v, K - 1);
            ti = __shfl_sync(kFull, i, K - 1);
        }
    }
};

// (max, sum exp(x - max)) of two parts; a part with max -inf is empty
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
    const float M = fmaxf(m, om);
    float S = 0.f;
    if (m > -INFINITY) S += s * expf(m - M);
    if (om > -INFINITY) S += os * expf(om - M);
    m = M;
    s = S;
}

// Merges the sorted lists of every warp of the CTA into warp 0's, pairwise in log2(warps) rounds (sv / si: [warps][32]
// shared scratch).
template <int kWarps>
__device__ void block_merge(WarpTopK& top, float (*sv)[32], int (*si)[32]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int s = 1; s < kWarps; s <<= 1) {
        sv[warp][lane] = top.v;
        si[warp][lane] = top.i;
        __syncthreads();
        if ((warp & (2 * s - 1)) == 0) top.merge_sorted(sv[warp + s][lane], si[warp + s][lane]);
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kChunkThreads) k_beam_chunk(const float* __restrict__ logits, int V,
                                                              const float* __restrict__ cum, int chunks, int per, int K,
                                                              float2* __restrict__ stats, BeamCand* __restrict__ lists) {
    pdl_trigger();
    pdl_wait();
    const int r = blockIdx.y, c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (!(cum[r] > -INFINITY)) return;   // dead row
    const int lo = c * per, hi = min(V, lo + per);
    const float* row = logits + (size_t)r * V;
    float m = -INFINITY, s = 0.f;
    WarpTopK top;
    top.init(K);
    for (int base = lo; base < hi; base += 4 * kChunkThreads) {   // uniform over the CTA
        float x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int idx = base + u * kChunkThreads + tid;
            x[u] = idx < hi ? row[idx] : -INFINITY;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const float xv = x[u];
            if (xv > m) {
                s = s * expf(m - xv) + 1.f;
                m = xv;
            } else if (xv > -INFINITY) {
                s += expf(xv - m);
            }
            top.offer(xv, base + u * kChunkThreads + tid, xv > -INFINITY && xv < INFINITY);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lse_merge(m, s, __shfl_xor_sync(kFull, m, o), __shfl_xor_sync(kFull, s, o));
    __shared__ float sm[kChunkThreads / 32], ss[kChunkThreads / 32];
    __shared__ float sv[kChunkThreads / 32][32];
    __shared__ int si[kChunkThreads / 32][32];
    if (lane == 0) {
        sm[warp] = m;
        ss[warp] = s;
    }
    block_merge<kChunkThreads / 32>(top, sv, si);
    if (warp == 0) {
        const size_t slot = (size_t)r * chunks + c;
        if (lane < K) lists[slot * K + lane] = BeamCand{top.v, top.i};
        if (lane == 0) {
            for (int w = 1; w < kChunkThreads / 32; ++w) lse_merge(m, s, sm[w], ss[w]);
            stats[slot] = make_float2(m, s);
        }
    }
}

__global__ void __launch_bounds__(kGroupThreads) k_beam_group(const float2* __restrict__ stats,
                                                              const BeamCand* __restrict__ lists, int chunks, int V,
                                                              const float* __restrict__ cum,
                                                              const int32_t* __restrict__ groups, int K,
                                                              int32_t* __restrict__ parent, int32_t* __restrict__ token,
                                                              float* __restrict__ score) {
    pdl_trigger();
    pdl_wait();
    constexpr int kWarps = kGroupThreads / 32;
    const int g = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int row0 = groups[2 * g], width = groups[2 * g + 1];
    __shared__ float s_max[kBeamMaxWidth], s_log[kBeamMaxWidth], s_cum[kBeamMaxWidth];
    // every live row's max and log(1e-20 + sum exp(x - max)) (beam_util.cu:30-41) from its chunks' statistics
    if (warp < width) {
        const float cr = cum[row0 + warp];
        float m = -INFINITY, s = 0.f;
        if (cr > -INFINITY)
            for (int c = lane; c < chunks; c += 32) {
                const float2 st = stats[(size_t)(row0 + warp) * chunks + c];
                lse_merge(m, s, st.x, st.y);
            }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lse_merge(m, s, __shfl_xor_sync(kFull, m, o), __shfl_xor_sync(kFull, s, o));
        if (lane == 0) {
            s_max[warp] = m;
            s_log[warp] = logf(1e-20f + s);
            s_cum[warp] = cr;
        }
    }
    __syncthreads();
    WarpTopK top;
    top.init(K);
    for (int l = warp; l < width * chunks; l += kWarps) {   // one chunk list per warp and pass
        const int j = l / chunks, c = l - j * chunks;
        const float cr = s_cum[j];
        if (!(cr > -INFINITY)) continue;   // dead row: its lists were never written
        BeamCand e{-INFINITY, INT_MAX};
        if (lane < K) e = lists[((size_t)(row0 + j) * chunks + c) * K + lane];
        // log_softmax_bias_without_temperature's order: x - max - log(sum) + bias
        const float sc = e.v - s_max[j] - s_log[j] + cr;
        const bool ok = lane < K && e.v > -INFINITY && sc > -INFINITY;
        top.offer(sc, ok ? j * V + e.i : INT_MAX, ok);
    }
    __shared__ float sv[kWarps][32];
    __shared__ int si[kWarps][32];
    block_merge<kWarps>(top, sv, si);
    if (warp == 0 && lane < K) {
        const bool ok = top.v > -INFINITY;
        parent[(size_t)g * K + lane] = ok ? top.i / V : -1;
        token[(size_t)g * K + lane] = ok ? top.i % V : -1;
        score[(size_t)g * K + lane] = ok ? top.v : -INFINITY;
    }
}

int beam_chunks(int R, int V) {
    int c = cdiv(kTargetCtas, R);
    const int by_len = cdiv(V, kMinChunk);
    if (c > by_len) c = by_len;
    if (c > kMaxChunks) c = kMaxChunks;
    return c < 1 ? 1 : c;
}

size_t align16(size_t b) { return (b + 15) / 16 * 16; }

// workspace: stats (R x chunks float2) | lists (R x chunks x K) | groups (2 R int32)
size_t ws_bytes_of(int R, int V, int K) {
    const size_t n = (size_t)R * beam_chunks(R, V);
    return align16(n * sizeof(float2)) + align16(n * K * sizeof(BeamCand)) + align16((size_t)2 * R * sizeof(int32_t));
}

}  // namespace

// host checks shared by zl_beam_topk and the driver's beam step (groups_host is a HOST array)
int beam_topk_check(int R, int V, const int32_t* groups_host, int G, int K) {
    ZL_CHECK_ARG(R > 0 && V > 0 && groups_host && G > 0 && G <= R);
    ZL_CHECK_ARG(K >= 1 && K <= kBeamMaxK);
    ZL_CHECK_SUPPORTED(V <= kBeamMaxVocab);
    int next = 0;   // the groups tile [0, R) in order
    for (int g = 0; g < G; ++g) {
        ZL_CHECK_ARG(groups_host[2 * g] == next);
        ZL_CHECK_ARG(groups_host[2 * g + 1] >= 1 && groups_host[2 * g + 1] <= kBeamMaxWidth);
        next += groups_host[2 * g + 1];
        ZL_CHECK_ARG(next <= R);
    }
    ZL_CHECK_ARG(next == R);
    return ZL_OK;
}

// the two launches over DEVICE groups (already checked); ws holds at least zl_beam_topk_workspace_bytes(R, V, K)
int beam_topk_launch(const float* logits, int R, int V, const float* cum, const int32_t* groups, int G, int K,
                     int32_t* parent, int32_t* token, float* score, void* ws, int pdl, cudaStream_t stream) {
    const int chunks = beam_chunks(R, V), per = cdiv(V, chunks);
    const size_t n = (size_t)R * chunks;
    float2* stats = static_cast<float2*>(ws);
    BeamCand* lists = reinterpret_cast<BeamCand*>(static_cast<char*>(ws) + align16(n * sizeof(float2)));
    ZL_CHECK_CUDA(launch(k_beam_chunk, dim3(chunks, R), dim3(kChunkThreads), 0, stream, pdl != 0, logits, V, cum, chunks,
                         per, K, stats, lists));
    ZL_CHECK_CUDA(launch(k_beam_group, dim3(G), dim3(kGroupThreads), 0, stream, pdl != 0, (const float2*)stats,
                         (const BeamCand*)lists, chunks, V, cum, groups, K, parent, token, score));
    return ZL_OK;
}

}  // namespace zl

using namespace zl;

extern "C" size_t zl_beam_topk_workspace_bytes(int R, int V, int K) {
    if (R <= 0 || V <= 0 || K <= 0) return 0;
    return ws_bytes_of(R, V, K);
}

extern "C" int zl_beam_topk(const float* logits, int R, int V, const float* cum, const int32_t* groups, int G, int K,
                            int32_t* parent, int32_t* token, float* score, void* ws, size_t ws_bytes, int pdl,
                            zl_stream_t stream) {
    ZL_CHECK_ARG(logits && cum && parent && token && score && ws);
    const int rc = beam_topk_check(R, V, groups, G, K);
    if (rc != ZL_OK) return rc;
    ZL_CHECK_ARG(ws_bytes >= ws_bytes_of(R, V, K));
    // the groups travel in the workspace's tail; a pageable source is staged before cudaMemcpyAsync returns
    const size_t n = (size_t)R * beam_chunks(R, V);
    int32_t* d_groups = reinterpret_cast<int32_t*>(static_cast<char*>(ws) + align16(n * sizeof(float2)) +
                                                   align16(n * K * sizeof(BeamCand)));
    ZL_CHECK_CUDA(cudaMemcpyAsync(d_groups, groups, sizeof(int32_t) * 2 * G, cudaMemcpyHostToDevice, stream));
    return beam_topk_launch(logits, R, V, cum, d_groups, G, K, parent, token, score, ws, pdl, stream);
}
