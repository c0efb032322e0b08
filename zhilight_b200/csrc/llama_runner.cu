// Host-side decode driver (C++): weights, KV buffers, the per-step kernel chain and its CUDA graph.
//
// Stands in for model::LLaMA::encode / EncoderLayer::forward / Attention::dynamic_batch_forward /
// FeedForward::forward at decode (reference src/model/llama.cpp:75-165, src/nn/block/block.cpp:86-143,
// src/nn/attention/attention.cpp:846-964, src/nn/feedforward/feedforward.cpp:113-137) and for the
// Int4GPTQ load pipeline (src/nn/linear/linear.cpp:1139-1244).  The reference launches ~12 kernels per
// layer with no graph; here a layer is 8 launches chained with programmatic dependent launch inside one
// CUDA graph per batch size.
#include "common.cuh"
#include "w4_layout.cuh"
#include "comm_dev.cuh"
#include "w4_params.h"

#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <utility>
#include <string>
#include <vector>

extern unsigned long long* g_w4_trace;   // debug timeline buffer (zl_w4_set_trace)

namespace {

// owning handles: device memory (cudaMalloc) and pinned host memory (cudaMallocHost)
struct CudaFree {
    void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
    void operator()(void* p) const { cudaFreeHost(p); }
};
template <typename T = void>
using dev_ptr = std::unique_ptr<T, CudaFree>;
template <typename T>
using host_ptr = std::unique_ptr<T, CudaFreeHost>;

struct Staged {
    dev_ptr<> ptr;
    int rows = 0, cols = 0, elem = 0;
};

struct W4Lin {
    dev_ptr<> packed;     // ZLW4  (fp16 HMMA kernels) -- only kept when some batch size needs it
    dev_ptr<> packed_i;   // ZLW4I (exact-integer IMMA kernel, small M)
    dev_ptr<> bias;
    int N = 0, K = 0;
    dev_ptr<int32_t> k_perm;   // act-order: the GEMM reads x[:, k_perm] (K int32); empty: sequential g_idx
};
struct DenseLin {
    dev_ptr<> w;
    dev_ptr<> bias;
    int N = 0, K = 0;
    // W8A8 (quant_type 2 / 7 / 10): 8-bit weights (N, K) + scales; w is released
    dev_ptr<> w8;
    dev_ptr<> w_scale;   // int8: (N) in the activation dtype (linear.cpp:541); fp8: (N) f32 rows;
                         // fp8 block: (N/128, K/128) f32 weight_scale_inv
    int w8_kind = -1;    // ZL_W8_INT8, ZL_W8_FP8_ROWS or kW8Block
};
constexpr int kW8Block = 10;   // QuantType 10 (Fp8Block): served by zl_fp8_block_gemm, not a zl_w8a8_gemm kind

struct Layer {
    dev_ptr<> ln_attn;
    dev_ptr<> ln_ff;
    W4Lin q_qkv, q_o, q_gu, q_down;
    DenseLin d_qkv, d_o, d_gu, d_down;
    dev_ptr<> kbuf;   // (max_batch, max_seq, Hkv, d): activation dtype, or uint8 codes at kv_int8
    dev_ptr<> vbuf;
    dev_ptr<void*> k_addrs;   // (max_batch)
    dev_ptr<void*> v_addrs;
    dev_ptr<> skbuf;          // kv_int8: (max_batch, max_seq, Hkv) fp32 scales
    dev_ptr<> svbuf;
    dev_ptr<void*> sk_addrs;  // (max_batch)
    dev_ptr<void*> sv_addrs;
};

}  // namespace

struct zl_llama {
    zl_llama_config_t cfg{};
    cudaStream_t stream = nullptr;
    std::map<std::string, Staged> staged;
    std::vector<Layer> layers;
    dev_ptr<> emb;
    dev_ptr<> lm_head_shard;        // untied lm_head (this rank's vocabulary rows)
    const void* lm_head = nullptr;  // lm_head_shard, or emb when tied
    dev_ptr<> ln_f;
    bool finalized = false;
    // local (per-rank) sizes
    int hq = 0, hkv = 0, ff = 0;
    // activations
    dev_ptr<> h2;   // second residual-stream buffer: the fused TP exchange ping-pongs between h and h2
    dev_ptr<> h, xn, qkv, q, ao, act, pend, gu;
    dev_ptr<float> logits;
    dev_ptr<float> cosb, sinb;
    dev_ptr<int32_t> d_tokens, d_pos, d_lens, d_next, d_iota;
    dev_ptr<> attn_ws;
    size_t attn_ws_bytes = 0;
    dev_ptr<> argmax_ws;
    host_ptr<int32_t> h_stage;   // tokens | pos | lens | next
    // zl_llama_set_state staging: pinned H2D copies read the host buffer when they EXECUTE, so a set_state -> step_device
    // loop that runs ahead of the GPU must not rewrite a slot whose copy is still queued: ring of slots, one event each
    static constexpr int kStageSlots = 8;
    host_ptr<int32_t> h_ring;    // [kStageSlots][2 * max_batch]
    cudaEvent_t ring_ev[kStageSlots] = {};
    bool ring_used[kStageSlots] = {};
    int ring_next = 0;
    // prefill keeps its own (token, position) arrays: the decode-state arrays d_tokens / d_pos of tasks 0..B-1 survive a
    // prefill that happens between two zl_llama_step_device calls (continuous batching)
    dev_ptr<int32_t> d_pf_tokens, d_pf_pos;
    const int32_t* cur_pos = nullptr;      // positions of the launch sequence being enqueued (d_pos or d_pf_pos)
    const int32_t* cur_tokens = nullptr;
    zl_comm_t* comm = nullptr;            // TP exchange (set by zl_llama_set_comm when tp_size > 1)
    int vshard = 0;                       // vocabulary rows of lm_head held by this rank
    dev_ptr<> cand;                       // [B] {float value, int index} local argmax candidates
    dev_ptr<> cand_all;                   // [tp][B] gathered candidates
    std::map<long long, cudaGraphExec_t> graphs;   // key = B * 2^32 + attention length bucket
    int cur_max_len = 0;                            // host-side upper bound of buf_lens (positions + 1)
    double weight_bytes = 0;
    int kernels_per_step = 0;
    // chunked prefill (cfg.prefill_chunk > 0): activation buffers hold tok_cap = max(max_batch, chunk) tokens
    int tok_cap = 0;
    // dual-stream chunked prefill (EncoderLayer::dual_stream_encode, block.cpp:205-441): compute stream = m->stream
    cudaStream_t reduce_stream = nullptr;
    cudaEvent_t ev_o[2] = {nullptr, nullptr}, ev_r1[2] = {nullptr, nullptr}, ev_dn[2] = {nullptr, nullptr},
                ev_r2[2] = {nullptr, nullptr};
    dev_ptr<> xq;              // W8A8: quantised activations of the Linear being run (tok_cap x max K bytes)
    dev_ptr<float> xs;         //       their scales (tok_cap; fp8 block: (max K/128, round_up(tok_cap, 4)))
    dev_ptr<int32_t> d_tb;     // token -> task map of the chunk being prefilled
    const int32_t* cur_tb = nullptr;   // token -> task map of the launch sequence being enqueued (d_iota at decode)
    dev_ptr<int8_t> d_mask;    // (chunk, max_seq) causal mask of the chunk
    // joined steps (zl_llama_step_joined): segments {task, row0, pos0, n} for zl_varlen_attention, then per emitting
    // segment its last row | its task | that row's position (max_batch each); h_join stages them with the tokens,
    // positions and token -> task map of the rows (tok_cap each) for the copies into d_pf_tokens / d_pf_pos / d_tb
    dev_ptr<int32_t> d_join;
    host_ptr<int32_t> h_join;
    dev_ptr<> xperm;           // act-order: activations permuted for the GEMM routes that cannot gather (tok_cap x max K)
    // sampling (zl_llama_set_sampling): per-task parameters and generated-token bitmaps on the device; samp_on[t] is set
    // while task t samples or has penalties, and the step then runs zl_sample instead of zl_argmax
    dev_ptr<zl_sample_params_t> d_sparams;   // (max_batch)
    dev_ptr<uint32_t> d_hist;                // (max_batch, hwords)
    int hwords = 0;
    std::vector<char> samp_on;
    // int8 KV cache: the rotated fp16 K / V rows of the launch sequence are staged in kv_stage (k: tok_cap x Hkv x d, then
    // v) and quantised into the cache from there.  A qkv GEMM with the RoPE / KV-append epilogue appends into the staging
    // rows as into the cache of one task: stage_addrs = {k rows, v rows}, token -> task map d_zeros, placement d_rowidx.
    dev_ptr<> kv_stage;
    dev_ptr<void*> stage_addrs;
    dev_ptr<int32_t> d_zeros, d_rowidx;      // (tok_cap): 0 ..., and 0, 1, 2, ...
    // the integer qkv GEMM's int8-cache epilogue: fp16 rows (16, 2, Hkv, d) and last-arriver counters (16, 2, Hkv), zero
    // between launches (every qkv GEMM of the model runs in stream order on the compute stream)
    dev_ptr<__half> kv8_rows;
    dev_ptr<uint32_t> kv8_cnt;
};

namespace {

using namespace zl;

#define RCHECK(expr)                \
    do {                            \
        int _rc = (expr);           \
        if (_rc != ZL_OK) return _rc; \
    } while (0)

template <typename T>
int dmalloc(dev_ptr<T>* p, size_t bytes) {
    void* raw = nullptr;
    ZL_CHECK_CUDA(cudaMalloc(&raw, bytes ? bytes : 16));
    p->reset(static_cast<T*>(raw));
    return ZL_OK;
}

__global__ void k_lens_from_pos(const int32_t* __restrict__ pos, int32_t* __restrict__ lens, int B,
                                unsigned long long* trace) {
    pdl_trigger();
    pdl_wait();
    if (trace && blockIdx.x == 0 && threadIdx.x == 0) trace[1] = globaltimer_ns();   // debug timeline: step start
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) lens[i] = pos[i] + 1;
}
__global__ void k_advance(int32_t* __restrict__ tokens, int32_t* __restrict__ pos, const int32_t* __restrict__ next,
                          int B, unsigned long long* trace) {
    if (trace && blockIdx.x == 0 && threadIdx.x == 0 && trace[2] == 0) trace[2] = globaltimer_ns();   // debug: first step end
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) {
        tokens[i] = next[i];
        pos[i] += 1;
    }
}
// prefill chunk setup: positions pos0.., token -> task map, the task's buffer length, and the causal mask
// mask[i][j] = j <= pos0 + i over len_buf = pos0 + n keys (attention_kernel.cu:434-489 mask contract, int8)
__global__ void k_prefill_setup(int32_t* __restrict__ pos, int32_t* __restrict__ tb, int32_t* __restrict__ lens,
                                int8_t* __restrict__ mask, int task, int pos0, int n) {
    const int len_buf = pos0 + n;
    for (int i = threadIdx.x + blockIdx.x * blockDim.x; i < n * len_buf; i += blockDim.x * gridDim.x) {
        const int qi = i / len_buf, j = i % len_buf;
        mask[i] = j <= pos0 + qi ? 1 : 0;
    }
    if (blockIdx.x == 0) {
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            pos[i] = pos0 + i;
            tb[i] = task;
        }
        if (threadIdx.x == 0) lens[task] = len_buf;
    }
}

// dst row i = src row idx[i] of a 16-bit (rows, D) matrix; grid = rows of dst
__global__ void k_gather_rows(const uint16_t* __restrict__ src, const int32_t* __restrict__ idx, uint16_t* __restrict__ dst,
                              int D) {
    const uint16_t* s = src + (size_t)idx[blockIdx.x] * D;
    uint16_t* o = dst + (size_t)blockIdx.x * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) o[i] = s[i];
}

template <typename T>
__global__ void k_f32_to_t(const float* __restrict__ in, T* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = from_f32<T>(in[i]);
}
__global__ void k_fill_from_scalar(float* __restrict__ dst, int n, const float* __restrict__ scalar) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = *scalar;
}
__global__ void k_and_u32(uint32_t* __restrict__ p, size_t n, uint32_t mask) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] &= mask;
}
__global__ void k_set_f32(float* p, float v) { *p = v; }
// in place: random u32 words -> f32 lo * (hi/lo)^u with u uniform in [0, 1)
__global__ void k_u32_to_log_uniform(uint32_t* __restrict__ p, int n, float lo, float hi) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = __float_as_uint(lo * powf(hi / lo, (float)(p[i] >> 8) * (1.f / 16777216.f)));
}
// synthetic symmetric checkpoints: a uniformly random nibble minus the fixed zero point 8 has mean -0.5, and with thousands
// of such weights per row every layer adds a common-mode offset to the residual stream that overflows fp16 after ~30
// layers (measured: NaN logits on the 32-layer model).  Nibble 0 -> 8 makes q - 8 symmetric around zero (-7 .. 7).
__global__ void k_recentre_nibbles(uint32_t* __restrict__ p, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const uint32_t w = p[i];
        const uint32_t zero = ~(w | (w >> 1) | (w >> 2) | (w >> 3)) & 0x11111111u;
        p[i] = w | (zero << 3);
    }
}

__global__ void k_iota(int32_t* p, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = i;
}
__global__ void k_ptr_table(void** tab, char* base, size_t stride, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) tab[i] = base + (size_t)i * stride;
}
__global__ void k_swiglu_row_map(int32_t* map, int F) {
    // packed row p: 16-row tile = 8 gate rows then the 8 matching up rows (source = [gate(F); up(F)])
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < 2 * F) {
        int tile = p >> 4, r = p & 15;
        map[p] = (r < 8) ? tile * 8 + r : F + tile * 8 + (r - 8);
    }
}

const Staged* find(const zl_llama* m, const std::string& name) {
    auto it = m->staged.find(name);
    return it == m->staged.end() ? nullptr : &it->second;
}

void drop(zl_llama* m, const std::string& name) { m->staged.erase(name); }

int fail_state(int line, const std::string& msg, int code = ZL_ERR_STATE) {
    zl_set_last_error(__FILE__, line, msg.c_str());
    return code;
}

// g_idx of a desc_act / act-order checkpoint is not k / group_size.  Like the reference (linear.cpp:1092-1094,
// 1145-1146), the load sorts it into a permutation -- argsort_cpu, a stable bucket sort of k by group
// (linear.cpp:1010-1028) -- gathers the weight rows with it (zl_gptq_shuffle with q_perm, make_sequential) and the GEMMs
// read x[:, perm] at run time.  perm is left empty when g_idx is missing or sequential: such Linears load exactly as before.
int g_idx_perm(zl_llama* m, const std::string& prefix, int K, std::vector<int32_t>* perm) {
    perm->clear();
    const Staged* gi = find(m, prefix + ".g_idx");
    if (!gi) return ZL_OK;
    if ((size_t)gi->rows * gi->cols != (size_t)K || gi->elem != 4)
        return fail_state(__LINE__, "ill-shaped g_idx for " + prefix + " (expected K int32)");
    const int g = m->cfg.group_size, G = K / g;
    std::vector<int32_t> host(K);
    ZL_CHECK_CUDA(cudaMemcpyAsync(host.data(), gi->ptr.get(), (size_t)K * 4, cudaMemcpyDeviceToHost, m->stream));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    bool sequential = true;
    for (int k = 0; k < K && sequential; ++k) sequential = host[k] == k / g;
    if (sequential) return ZL_OK;
    if (m->cfg.tp_size > 1) {
        return fail_state(__LINE__, "act-order (desc_act) GPTQ checkpoint (" + prefix + ".g_idx) with tp_size > 1: a rank's "
                                        "o_proj input shard does not hold the columns its permuted K shard needs",
                          ZL_ERR_UNSUPPORTED);
    }
    // K entries, none past the last group and none in a full group: every group has exactly g members
    std::vector<int> count(G, 0);
    perm->assign(K, 0);
    for (int k = 0; k < K; ++k) {
        const int grp = host[k];
        if (grp < 0 || grp >= G || count[grp] >= g) {
            perm->clear();
            return fail_state(__LINE__, "malformed g_idx for " + prefix + ": every group of " + std::to_string(g) +
                                            " columns must appear exactly " + std::to_string(g) + " times",
                              ZL_ERR_INVALID_ARG);
        }
        (*perm)[grp * g + count[grp]++] = k;
    }
    return ZL_OK;
}

// presence, shape and element size of one Linear's GPTQ/AWQ tensors
int check_quant_tensors(zl_llama* m, const std::string& prefix, int K, int N) {
    const Staged* qw = find(m, prefix + ".qweight");
    const Staged* qz = find(m, prefix + ".qzeros");
    const Staged* sc = find(m, prefix + ".scales");
    if (!qw || !qz || !sc) return fail_state(__LINE__, "missing GPTQ tensors for " + prefix);
    const int G = K / m->cfg.group_size;
    const bool awq = m->cfg.quant_type == 6;
    const bool qw_ok = awq ? (qw->rows == K && qw->cols == N / 8) : (qw->rows == K / 8 && qw->cols == N);
    if (!qw_ok || qw->elem != 4) return fail_state(__LINE__, "ill-shaped qweight for " + prefix, ZL_ERR_INVALID_ARG);
    if (qz->rows != G || qz->cols != N / 8 || qz->elem != 4)
        return fail_state(__LINE__, "ill-shaped qzeros for " + prefix + " (expected (K/g, N/8) int32)", ZL_ERR_INVALID_ARG);
    if (sc->rows != G || sc->cols != N || sc->elem != 2)
        return fail_state(__LINE__, "ill-shaped scales for " + prefix + " (expected (K/g, N) fp16)", ZL_ERR_INVALID_ARG);
    return ZL_OK;
}

// HF GPTQ/AWQ tensors of one Linear -> reference k-major tensors written at row offset n_off of the fused
// k-major buffers (linear.cpp:1139-1160 preprocess_weight + 1085-1099 transpose_weight).  q_perm (device, K) or nullptr:
// the act-order permutation the weight rows are gathered with.
int to_k_major(zl_llama* m, const std::string& prefix, int K, int N, uint32_t* qw_km, uint8_t* qz_km, __half* sc_km,
               int n_off, const int32_t* q_perm = nullptr) {
    // every shape / element size is validated BEFORE the first kernel touches the tensors (in-place transforms below)
    RCHECK(check_quant_tensors(m, prefix, K, N));
    const Staged* qw = find(m, prefix + ".qweight");
    const Staged* qz = find(m, prefix + ".qzeros");
    const Staged* sc = find(m, prefix + ".scales");
    const int G = K / m->cfg.group_size;
    const bool awq = m->cfg.quant_type == 6;
    cudaStream_t st = m->stream;
    uint32_t* qz_p = static_cast<uint32_t*>(qz->ptr.get());
    dev_ptr<uint32_t> tmp;   // AWQ: the un-shuffled weight; act-order GPTQ: the gather's scratch
    uint32_t* w_kn = nullptr;   // (K/8, N)
    if (awq) {
        RCHECK(dmalloc(&tmp, (size_t)(K / 8) * N * 4));
        w_kn = tmp.get();
        RCHECK(zl_awq_shuffle(static_cast<const uint32_t*>(qw->ptr.get()), w_kn, K, N, 1, st));
        RCHECK(zl_awq_un_shuffle(qz_p, G, N / 8, st));
    } else {
        w_kn = static_cast<uint32_t*>(qw->ptr.get());
        if (q_perm) RCHECK(dmalloc(&tmp, (size_t)(K / 8) * N * 4));
        RCHECK(zl_gptq_shuffle(w_kn, q_perm, tmp.get(), K, N, st));
        RCHECK(zl_gptq_increase_zero(qz_p, (size_t)G * (N / 8), st));
    }
    dev_ptr<uint8_t> z8;   // (G, N)
    RCHECK(dmalloc(&z8, (size_t)G * N));
    RCHECK(zl_q4_to_q8(qz_p, z8.get(), (size_t)G * (N / 8), st));
    // transposes straight into the fused buffers (row offset n_off)
    RCHECK(zl_transpose_2d(w_kn, qw_km + (size_t)n_off * (K / 8), K / 8, N, 4, st));
    RCHECK(zl_transpose_2d(z8.get(), qz_km + (size_t)n_off * G, G, N, 1, st));
    RCHECK(zl_transpose_2d(sc->ptr.get(), sc_km + (size_t)n_off * G, G, N, 2, st));
    ZL_CHECK_CUDA(cudaStreamSynchronize(st));
    return ZL_OK;
}

// ZL_W4_FORCE_HALF (A/B baseline): every W4 GEMM takes the fp16 mma.sync route.  Read once per process.
bool force_half() {
    static const bool v = getenv("ZL_W4_FORCE_HALF") != nullptr;
    return v;
}

// The kernel that serves a W4 Linear at B rows: 3 exact-integer, 4 wgmma, 0 fp16 mma.sync.
int route_of(const W4Lin& w, int B) { return w.packed_i && !force_half() ? zl_w4_int_layout_route(B, w.N, w.K) : 0; }

// The (N) fp16 bias of Linears fused along N: zeros, with each present `prefix.bias` at its row offset.  *out stays
// empty when none has one.  Every staged bias is checked before the first copy.
int build_bias(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, dev_ptr<>* out) {
    int N = 0;
    bool any = false;
    for (size_t i = 0; i < prefixes.size(); ++i) {
        const Staged* b = find(m, prefixes[i] + ".bias");
        if (b && ((size_t)b->rows * b->cols != (size_t)ns[i] || b->elem != 2))
            return fail_state(__LINE__, "ill-shaped bias " + prefixes[i] + ".bias (expected " + std::to_string(ns[i]) +
                                            " fp16)", ZL_ERR_INVALID_ARG);
        any |= b != nullptr;
        N += ns[i];
    }
    if (!any) return ZL_OK;
    RCHECK(dmalloc(out, (size_t)N * 2));
    ZL_CHECK_CUDA(cudaMemsetAsync(out->get(), 0, (size_t)N * 2, m->stream));
    int off = 0;
    for (size_t i = 0; i < prefixes.size(); ++i) {
        if (const Staged* b = find(m, prefixes[i] + ".bias"))
            ZL_CHECK_CUDA(cudaMemcpyAsync((char*)out->get() + (size_t)off * 2, b->ptr.get(), (size_t)ns[i] * 2,
                                          cudaMemcpyDeviceToDevice, m->stream));
        off += ns[i];
    }
    return ZL_OK;
}

// out_rows (swiglu only, act-order w_out): w_out's permutation, folded into the gate / up row order.
// keep_perm = false: the weight rows are sequentialised but the GEMM runs without k_perm (its producer wrote x permuted).
int build_w4(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, int K, bool swiglu,
             W4Lin* out, bool qkv_rope = false, const std::vector<int32_t>* out_rows = nullptr, bool keep_perm = true) {
    int N = 0;
    for (int n : ns) N += n;
    const int G = K / m->cfg.group_size;
    // act-order: Linears fused along N share their input, so they must share its permutation.  Real checkpoints give
    // q / k / v (and gate / up) the same g_idx: their GPTQ Hessian is that of the same input.
    std::vector<int32_t> perm, other;
    for (size_t i = 0; i < prefixes.size(); ++i) {
        RCHECK(check_quant_tensors(m, prefixes[i], K, ns[i]));   // the errors of a Linear keep their order
        RCHECK(g_idx_perm(m, prefixes[i], K, i ? &other : &perm));
        if (i && other != perm)
            return fail_state(__LINE__, "act-order g_idx of " + prefixes[i] + " differs from " + prefixes[0] +
                                            ": Linears fused on one input need one permutation",
                              ZL_ERR_UNSUPPORTED);
    }
    if (!perm.empty() && m->cfg.quant_type == 6)
        return fail_state(__LINE__, "non-sequential g_idx on an AWQ checkpoint: " + prefixes[0], ZL_ERR_UNSUPPORTED);
    dev_ptr<int32_t> perm_tmp;   // keep_perm = false: the permutation only serves the weight gather
    dev_ptr<int32_t>& d_perm = keep_perm ? out->k_perm : perm_tmp;
    if (!perm.empty()) {
        RCHECK(dmalloc(&d_perm, (size_t)K * 4));
        ZL_CHECK_CUDA(cudaMemcpyAsync(d_perm.get(), perm.data(), (size_t)K * 4, cudaMemcpyHostToDevice, m->stream));
    }
    dev_ptr<uint32_t> qw_km;
    dev_ptr<uint8_t> qz_km;
    dev_ptr<__half> sc_km;
    RCHECK(dmalloc(&qw_km, (size_t)N * (K / 8) * 4));
    RCHECK(dmalloc(&qz_km, (size_t)N * G));
    RCHECK(dmalloc(&sc_km, (size_t)N * G * 2));
    int off = 0;
    for (size_t i = 0; i < prefixes.size(); ++i) {
        RCHECK(to_k_major(m, prefixes[i], K, ns[i], qw_km.get(), qz_km.get(), sc_km.get(), off, d_perm.get()));
        off += ns[i];
    }
    dev_ptr<int32_t> row_map;
    if (swiglu && out_rows && !out_rows->empty()) {
        // PERMUTE_FF_UP_OUT (linear.cpp:1168-1210): gate row j and up row j of the pack (still interleaved 8 + 8 per
        // 16-row tile for the SwiGLU epilogue) come from source row out_rows[j], so the SwiGLU output is already in
        // w_out's sequentialised k order and the down GEMM needs no permute
        const int F = N / 2;
        std::vector<int32_t> h(N);
        for (int p = 0; p < N; ++p) {
            const int r = p & 15;
            h[p] = (r < 8 ? 0 : F) + (*out_rows)[(p >> 4) * 8 + (r & 7)];
        }
        RCHECK(dmalloc(&row_map, (size_t)N * 4));
        ZL_CHECK_CUDA(cudaMemcpyAsync(row_map.get(), h.data(), (size_t)N * 4, cudaMemcpyHostToDevice, m->stream));
        ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));   // h is pageable and goes out of scope
    } else if (swiglu) {
        RCHECK(dmalloc(&row_map, (size_t)N * 4));
        k_swiglu_row_map<<<cdiv(N, 256), 256, 0, m->stream>>>(row_map.get(), N / 2);
        ZL_CHECK_LAUNCH();
    } else if (qkv_rope) {
        RCHECK(dmalloc(&row_map, (size_t)N * 4));
        RCHECK(zl_qkv_rope_row_map(row_map.get(), N / m->cfg.dim_head, m->cfg.dim_head, m->stream));
    }
    const size_t pbytes = zl_w4_packed_bytes(N, K, m->cfg.group_size);
    ZL_CHECK_SUPPORTED(pbytes > 0);
    // the ZLW4I layout serves the exact-integer kernel (M <= 16 when its staged activations fit) and the wgmma kernel
    // (any M, N % 128 == 0); the fp16 mma.sync layout is only materialised when some launch size has neither
    const int m_max = m->cfg.prefill_chunk > m->cfg.max_batch ? m->cfg.prefill_chunk : m->cfg.max_batch;
    bool need_half = force_half();
    for (int mm = 1; mm <= (m_max < 17 ? m_max : 17); ++mm)
        if (!zl_w4_int_layout_route(mm, N, K)) need_half = true;
    RCHECK(dmalloc(&out->packed_i, pbytes));
    RCHECK(zl_w4_pack_v(qw_km.get(), qz_km.get(), sc_km.get(), row_map.get(), out->packed_i.get(), N, K,
                        m->cfg.group_size, m->cfg.sym, 1, m->stream));
    if (need_half) {
        RCHECK(dmalloc(&out->packed, pbytes));
        RCHECK(zl_w4_pack_v(qw_km.get(), qz_km.get(), sc_km.get(), row_map.get(), out->packed.get(), N, K,
                            m->cfg.group_size, m->cfg.sym, 0, m->stream));
    }
    if (!swiglu) {
        RCHECK(build_bias(m, prefixes, ns, &out->bias));
        if (out->bias && row_map) {   // the fused epilogues index bias by packed row
            dev_ptr<> pb;
            RCHECK(dmalloc(&pb, (size_t)N * 2));
            RCHECK(zl_gather_rows_16(out->bias.get(), row_map.get(), pb.get(), N, m->stream));
            ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
            out->bias = std::move(pb);
        }
    }
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    for (auto& p : prefixes) {
        drop(m, p + ".qweight");
        drop(m, p + ".qzeros");
        drop(m, p + ".scales");
        drop(m, p + ".g_idx");
        drop(m, p + ".bias");
    }
    out->N = N;
    out->K = K;
    m->weight_bytes += (double)pbytes;
    return ZL_OK;
}

int build_dense(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, int K,
                DenseLin* out) {
    int N = 0;
    for (int n : ns) N += n;
    RCHECK(dmalloc(&out->w, (size_t)N * K * 2));
    int off = 0;
    for (size_t i = 0; i < prefixes.size(); ++i) {
        const Staged* w = find(m, prefixes[i] + ".weight");
        if (!w || w->rows != ns[i] || w->cols != K || w->elem != 2) {
            zl_set_last_error(__FILE__, __LINE__, ("missing/ill-shaped dense weight " + prefixes[i]).c_str());
            return ZL_ERR_STATE;
        }
        ZL_CHECK_CUDA(cudaMemcpyAsync((char*)out->w.get() + (size_t)off * K * 2, w->ptr.get(), (size_t)ns[i] * K * 2,
                                      cudaMemcpyDeviceToDevice, m->stream));
        off += ns[i];
    }
    RCHECK(build_bias(m, prefixes, ns, &out->bias));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    for (auto& p : prefixes) {
        drop(m, p + ".weight");
        drop(m, p + ".bias");
    }
    out->N = N;
    out->K = K;
    m->weight_bytes += (double)N * K * 2;
    return ZL_OK;
}

// quant_type 2 (AutoInt8, linear.cpp:521-550): the fp weight is quantised per output row at load with the same kernel
// as the activations; the scale is kept in the activation dtype (functions::typecast, linear.cpp:541).
int dense_to_int8(zl_llama* m, DenseLin* d) {
    const auto& c = m->cfg;
    dev_ptr<float> sf;
    RCHECK(dmalloc(&d->w8, (size_t)d->N * d->K));
    RCHECK(dmalloc(&sf, (size_t)d->N * 4));
    RCHECK(dmalloc(&d->w_scale, (size_t)d->N * 2));
    RCHECK(zl_int8_quant_per_token(d->w.get(), d->K, d->w8.get(), sf.get(), d->N, d->K, c.dtype, 0, m->stream));
    if (c.dtype == ZL_F16)
        k_f32_to_t<__half><<<cdiv(d->N, 256), 256, 0, m->stream>>>(sf.get(), static_cast<__half*>(d->w_scale.get()), d->N);
    else
        k_f32_to_t<__nv_bfloat16><<<cdiv(d->N, 256), 256, 0, m->stream>>>(
            sf.get(), static_cast<__nv_bfloat16*>(d->w_scale.get()), d->N);
    ZL_CHECK_LAUNCH();
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    d->w.reset();
    d->w8_kind = ZL_W8_INT8;
    m->weight_bytes += (double)d->N * d->K + (double)d->N * 2 - (double)d->N * d->K * 2;
    return ZL_OK;
}

// quant_type 7 (Fp8Linear, linear.cpp:1612-1695): e4m3 weights + one f32 weight_scale per Linear.  Projections that
// share an input are fused along N with their scalar scales expanded to one scale per output row.
int build_fp8(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, int K, DenseLin* out) {
    int N = 0;
    for (int n : ns) N += n;
    RCHECK(dmalloc(&out->w8, (size_t)N * K));
    RCHECK(dmalloc(&out->w_scale, (size_t)N * 4));
    int off = 0;
    for (size_t i = 0; i < prefixes.size(); ++i) {
        const Staged* w = find(m, prefixes[i] + ".weight");
        const Staged* ws = find(m, prefixes[i] + ".weight_scale");
        if (!w || w->rows != ns[i] || w->cols != K || w->elem != 1 || !ws || ws->elem != 4) {
            zl_set_last_error(__FILE__, __LINE__, ("missing/ill-shaped fp8 weight or weight_scale " + prefixes[i]).c_str());
            return ZL_ERR_STATE;
        }
        ZL_CHECK_CUDA(cudaMemcpyAsync((char*)out->w8.get() + (size_t)off * K, w->ptr.get(), (size_t)ns[i] * K,
                                      cudaMemcpyDeviceToDevice, m->stream));
        k_fill_from_scalar<<<cdiv(ns[i], 256), 256, 0, m->stream>>>(static_cast<float*>(out->w_scale.get()) + off, ns[i],
                                                                     static_cast<const float*>(ws->ptr.get()));
        ZL_CHECK_LAUNCH();
        off += ns[i];
    }
    RCHECK(build_bias(m, prefixes, ns, &out->bias));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    for (auto& p : prefixes) {
        drop(m, p + ".weight");
        drop(m, p + ".weight_scale");
        drop(m, p + ".bias");
    }
    out->N = N;
    out->K = K;
    out->w8_kind = ZL_W8_FP8_ROWS;
    m->weight_bytes += (double)N * K + (double)N * 4;
    return ZL_OK;
}

// quant_type 10 (Fp8Block, linear.cpp:1697-1960): e4m3 weights + weight_scale_inv with one f32 per 128x128 block.
// Projections that share an input are fused along N by concatenating both their weight rows and their scale rows,
// which needs every part's N to be a multiple of 128.  Fp8Block has no bias (set_has_bias throws).
int build_fp8_block(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, int K,
                    DenseLin* out) {
    int N = 0;
    for (int n : ns) N += n;
    if (K % 128 != 0 || (prefixes.size() > 1 && N % 128 != 0))
        return fail_state(__LINE__, "fp8 block weights need K % 128 == 0 and every fused part's N % 128 == 0",
                          ZL_ERR_UNSUPPORTED);
    for (size_t i = 0; i < prefixes.size(); ++i) {
        if (prefixes.size() > 1 && ns[i] % 128 != 0)
            return fail_state(__LINE__, "fp8 block weights: fused part " + prefixes[i] + " has N % 128 != 0",
                              ZL_ERR_UNSUPPORTED);
        if (find(m, prefixes[i] + ".bias"))
            return fail_state(__LINE__, "fp8 block Linear " + prefixes[i] + " has a bias (Fp8Block has none)",
                              ZL_ERR_UNSUPPORTED);
    }
    const int KB = K / 128, NB = (N + 127) / 128;
    RCHECK(dmalloc(&out->w8, (size_t)N * K));
    RCHECK(dmalloc(&out->w_scale, (size_t)NB * KB * 4));
    int off = 0;
    for (size_t i = 0; i < prefixes.size(); ++i) {
        const Staged* w = find(m, prefixes[i] + ".weight");
        const Staged* ws = find(m, prefixes[i] + ".weight_scale_inv");
        const int nb = (ns[i] + 127) / 128;
        if (!w || w->rows != ns[i] || w->cols != K || w->elem != 1 || !ws || ws->elem != 4 || ws->rows != nb ||
            ws->cols != KB) {
            zl_set_last_error(__FILE__, __LINE__,
                              ("missing/ill-shaped fp8 block weight or weight_scale_inv " + prefixes[i]).c_str());
            return ZL_ERR_STATE;
        }
        ZL_CHECK_CUDA(cudaMemcpyAsync((char*)out->w8.get() + (size_t)off * K, w->ptr.get(), (size_t)ns[i] * K,
                                      cudaMemcpyDeviceToDevice, m->stream));
        ZL_CHECK_CUDA(cudaMemcpyAsync((char*)out->w_scale.get() + (size_t)(off / 128) * KB * 4, ws->ptr.get(),
                                      (size_t)nb * KB * 4, cudaMemcpyDeviceToDevice, m->stream));
        off += ns[i];
    }
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    for (auto& p : prefixes) {
        drop(m, p + ".weight");
        drop(m, p + ".weight_scale_inv");
    }
    out->N = N;
    out->K = K;
    out->w8_kind = kW8Block;
    m->weight_bytes += (double)N * K + (double)NB * KB * 4;
    return ZL_OK;
}

int take_vector(zl_llama* m, const std::string& name, int n, dev_ptr<>* out) {
    auto it = m->staged.find(name);
    if (it == m->staged.end() || (size_t)it->second.rows * it->second.cols != (size_t)n || it->second.elem != 2) {
        zl_set_last_error(__FILE__, __LINE__, ("missing/ill-shaped tensor " + name).c_str());
        return ZL_ERR_STATE;
    }
    *out = std::move(it->second.ptr);
    m->staged.erase(it);
    m->weight_bytes += (double)n * 2;
    return ZL_OK;
}

int finalize_layer(zl_llama* m, int l) {
    const auto& c = m->cfg;
    Layer& L = m->layers[l];
    const std::string p = "layers." + std::to_string(l) + ".";
    const int D = c.dim_model, d = c.dim_head;
    RCHECK(take_vector(m, p + "ln_attn.weight", D, &L.ln_attn));
    RCHECK(take_vector(m, p + "ln_ff.weight", D, &L.ln_ff));
    const std::vector<std::string> qkv = {p + "attn.project_q", p + "attn.project_k", p + "attn.project_v"};
    const std::vector<int> qkv_n = {m->hq * d, m->hkv * d, m->hkv * d};
    const std::vector<std::string> gu = {p + "ff.w_in", p + "ff.w_gated"};
    const std::vector<int> gu_n = {m->ff, m->ff};
    if (c.quant_type == 5 || c.quant_type == 6) {
        // act-order w_out: its permutation orders the gate / up rows, so down runs without one.  A bad w_out g_idx is
        // reported by its own build_w4 below, after the errors of the Linears built before it.
        std::vector<int32_t> down_perm;
        if (g_idx_perm(m, p + "ff.w_out", m->ff, &down_perm) != ZL_OK) down_perm.clear();
        RCHECK(build_w4(m, qkv, qkv_n, D, false, &L.q_qkv, c.fuse >= 2));
        RCHECK(build_w4(m, {p + "attn.attn_out"}, {D}, m->hq * d, false, &L.q_o));
        RCHECK(build_w4(m, gu, gu_n, D, true, &L.q_gu, false, &down_perm));
        RCHECK(build_w4(m, {p + "ff.w_out"}, {D}, m->ff, false, &L.q_down, false, nullptr, false));
    } else if (c.quant_type == 7) {
        RCHECK(build_fp8(m, qkv, qkv_n, D, &L.d_qkv));
        RCHECK(build_fp8(m, {p + "attn.attn_out"}, {D}, m->hq * d, &L.d_o));
        RCHECK(build_fp8(m, gu, gu_n, D, &L.d_gu));
        RCHECK(build_fp8(m, {p + "ff.w_out"}, {D}, m->ff, &L.d_down));
    } else if (c.quant_type == 10) {
        RCHECK(build_fp8_block(m, qkv, qkv_n, D, &L.d_qkv));
        RCHECK(build_fp8_block(m, {p + "attn.attn_out"}, {D}, m->hq * d, &L.d_o));
        RCHECK(build_fp8_block(m, gu, gu_n, D, &L.d_gu));
        RCHECK(build_fp8_block(m, {p + "ff.w_out"}, {D}, m->ff, &L.d_down));
    } else {
        RCHECK(build_dense(m, qkv, qkv_n, D, &L.d_qkv));
        RCHECK(build_dense(m, {p + "attn.attn_out"}, {D}, m->hq * d, &L.d_o));
        RCHECK(build_dense(m, gu, gu_n, D, &L.d_gu));
        RCHECK(build_dense(m, {p + "ff.w_out"}, {D}, m->ff, &L.d_down));
        if (c.quant_type == 2)
            for (DenseLin* dl : {&L.d_qkv, &L.d_o, &L.d_gu, &L.d_down}) RCHECK(dense_to_int8(m, dl));
    }
    return ZL_OK;
}

int finalize_globals(zl_llama* m) {
    const auto& c = m->cfg;
    RCHECK(take_vector(m, "token_embedding.weight", c.vocab_size * c.dim_model, &m->emb));
    m->weight_bytes -= (double)c.vocab_size * c.dim_model * 2;   // the embedding table is gathered, not streamed
    RCHECK(take_vector(m, "output_layernorm.weight", c.dim_model, &m->ln_f));
    if (find(m, "lm_head.weight")) {
        RCHECK(take_vector(m, "lm_head.weight", m->vshard * c.dim_model, &m->lm_head_shard));   // vocab-parallel shard
        m->lm_head = m->lm_head_shard.get();
    } else {
        ZL_CHECK_SUPPORTED(c.tp_size == 1);   // tied lm_head is only wired for a single rank
        m->lm_head = m->emb.get();   // tied (Llama-3.2-1B)
        m->weight_bytes += (double)c.vocab_size * c.dim_model * 2;
    }
    return ZL_OK;
}

int alloc_runtime(zl_llama* m) {
    const auto& c = m->cfg;
    const int B = c.max_batch, D = c.dim_model, d = c.dim_head;
    // bytes per task: codes (1 byte per value) + one fp32 scale per (token, kv head) at kv_int8, else 2 bytes per value
    const size_t kv_task = (size_t)c.max_seq * m->hkv * d * (c.kv_int8 ? 1 : 2);
    const size_t sc_task = (size_t)c.max_seq * m->hkv * 4;
    // never-written rows must be finite: masked keys still multiply their V rows by an exact 0, and with the dual-stream
    // prefill one half's attention sees the other half's rows before they are appended.  Zero codes with zero scales
    // decode to 0.
    auto cache = [&](dev_ptr<>* buf, dev_ptr<void*>* tab, size_t per_task) -> int {
        RCHECK(dmalloc(buf, per_task * B));
        ZL_CHECK_CUDA(cudaMemsetAsync(buf->get(), 0, per_task * B, m->stream));
        RCHECK(dmalloc(tab, sizeof(void*) * B));
        k_ptr_table<<<cdiv(B, 256), 256, 0, m->stream>>>(tab->get(), (char*)buf->get(), per_task, B);
        ZL_CHECK_LAUNCH();
        return ZL_OK;
    };
    for (auto& L : m->layers) {
        RCHECK(cache(&L.kbuf, &L.k_addrs, kv_task));
        RCHECK(cache(&L.vbuf, &L.v_addrs, kv_task));
        if (c.kv_int8) {
            RCHECK(cache(&L.skbuf, &L.sk_addrs, sc_task));
            RCHECK(cache(&L.svbuf, &L.sv_addrs, sc_task));
        }
    }
    const int T = c.prefill_chunk > B ? c.prefill_chunk : B;   // tokens per launch: decode batch or prefill chunk
    m->tok_cap = T;
    if (c.kv_int8) {
        const size_t rows_bytes = (size_t)T * m->hkv * d * 2;
        RCHECK(dmalloc(&m->kv_stage, 2 * rows_bytes));
        RCHECK(dmalloc(&m->stage_addrs, sizeof(void*) * 2));
        k_ptr_table<<<1, 32, 0, m->stream>>>(m->stage_addrs.get(), (char*)m->kv_stage.get(), rows_bytes, 2);
        RCHECK(dmalloc(&m->d_zeros, (size_t)T * 4));
        ZL_CHECK_CUDA(cudaMemsetAsync(m->d_zeros.get(), 0, (size_t)T * 4, m->stream));
        RCHECK(dmalloc(&m->d_rowidx, (size_t)T * 4));
        k_iota<<<cdiv(T, 256), 256, 0, m->stream>>>(m->d_rowidx.get(), T);
        ZL_CHECK_LAUNCH();
        RCHECK(dmalloc(&m->kv8_rows, (size_t)16 * 2 * m->hkv * d * 2));
        RCHECK(dmalloc(&m->kv8_cnt, (size_t)16 * 2 * m->hkv * 4));
        ZL_CHECK_CUDA(cudaMemsetAsync(m->kv8_cnt.get(), 0, (size_t)16 * 2 * m->hkv * 4, m->stream));
    }
    RCHECK(dmalloc(&m->h, (size_t)T * D * 2));
    RCHECK(dmalloc(&m->xn, (size_t)T * D * 2));
    if (c.tp_size > 1) RCHECK(dmalloc(&m->h2, (size_t)T * D * 2));
    RCHECK(dmalloc(&m->pend, (size_t)T * D * 2));
    RCHECK(dmalloc(&m->qkv, (size_t)T * (m->hq + 2 * m->hkv) * d * 2));
    RCHECK(dmalloc(&m->q, (size_t)T * m->hq * d * 2));
    RCHECK(dmalloc(&m->ao, (size_t)T * m->hq * d * 2));
    RCHECK(dmalloc(&m->gu, (size_t)T * 2 * m->ff * 2));
    RCHECK(dmalloc(&m->act, (size_t)T * m->ff * 2));
    bool act_order = false;
    for (const auto& L : m->layers) act_order |= L.q_qkv.k_perm || L.q_o.k_perm || L.q_gu.k_perm;
    if (act_order) RCHECK(dmalloc(&m->xperm, (size_t)T * (D > m->hq * d ? D : m->hq * d) * 2));
    RCHECK(dmalloc(&m->logits, (size_t)B * c.vocab_size * 4));
    RCHECK(dmalloc(&m->cand, (size_t)((B * 8 + 15) / 16) * 16));
    RCHECK(dmalloc(&m->cand_all, (size_t)((B * 8 + 15) / 16) * 16 * c.tp_size));
    RCHECK(dmalloc(&m->cosb, (size_t)T * d * 4));
    RCHECK(dmalloc(&m->sinb, (size_t)T * d * 4));
    RCHECK(dmalloc(&m->d_tokens, B * 4));
    RCHECK(dmalloc(&m->d_pos, B * 4));
    RCHECK(dmalloc(&m->d_lens, B * 4));
    if (c.quant_type == 2 || c.quant_type == 7 || c.quant_type == 10) {
        int kmax = D > m->ff ? D : m->ff;
        kmax = kmax > m->hq * d ? kmax : m->hq * d;
        RCHECK(dmalloc(&m->xq, (size_t)T * kmax));
        // fp8 block: one scale per (token, 128 columns), column-major with leading dimension round_up(tokens, 4)
        RCHECK(dmalloc(&m->xs, c.quant_type == 10 ? (size_t)(kmax / 128 + 1) * ((T + 3) / 4 * 4) * 4 : (size_t)T * 4));
    }
    if (c.prefill_chunk > 0) {
        RCHECK(dmalloc(&m->d_tb, T * 4));
        RCHECK(dmalloc(&m->d_pf_tokens, T * 4));
        RCHECK(dmalloc(&m->d_pf_pos, T * 4));
        RCHECK(dmalloc(&m->d_mask, (size_t)c.prefill_chunk * c.max_seq));
        RCHECK(dmalloc(&m->d_join, (size_t)7 * B * 4));
        int32_t* hj = nullptr;
        ZL_CHECK_CUDA(cudaMallocHost((void**)&hj, sizeof(int32_t) * ((size_t)3 * T + 7 * B)));
        m->h_join.reset(hj);
    }
    RCHECK(dmalloc(&m->d_next, B * 4));
    RCHECK(dmalloc(&m->d_iota, B * 4));
    k_iota<<<cdiv(B, 256), 256, 0, m->stream>>>(m->d_iota.get(), B);
    ZL_CHECK_LAUNCH();
    // also bounds zl_decode_attention_kv8: it splits the keys into at most 64 pieces (kA8MaxSplits, at least
    // cdiv(max_len, 1024)) over B * len_q <= T query rows, and this reserves T * Hq * max(64, cdiv(max_seq, 1024)) pieces
    m->attn_ws_bytes = zl_decode_attention_workspace_bytes(T, 1, m->hq, d, c.max_seq);
    if (c.prefill_chunk > 0) {   // joined steps: zl_varlen_attention over at most T rows of at most max_seq keys
        const size_t va = zl_varlen_attention_workspace_bytes(T, 1, m->hq, d, c.max_seq);
        if (va > m->attn_ws_bytes) m->attn_ws_bytes = va;
    }
    RCHECK(dmalloc(&m->attn_ws, m->attn_ws_bytes));
    RCHECK(dmalloc(&m->argmax_ws, zl_argmax_workspace_bytes(B)));
    m->hwords = cdiv(m->vshard, 32);
    RCHECK(dmalloc(&m->d_hist, (size_t)B * m->hwords * 4));
    ZL_CHECK_CUDA(cudaMemsetAsync(m->d_hist.get(), 0, (size_t)B * m->hwords * 4, m->stream));
    RCHECK(dmalloc(&m->d_sparams, sizeof(zl_sample_params_t) * B));
    {
        const zl_sample_params_t greedy{0.f, 1.f, 1.f, 0.f, 0, 0};
        std::vector<zl_sample_params_t> init(B, greedy);
        ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_sparams.get(), init.data(), sizeof(zl_sample_params_t) * B, cudaMemcpyHostToDevice,
                                      m->stream));
        ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));   // `init` is pageable and goes out of scope
    }
    m->samp_on.assign(B, 0);
    int32_t *stage = nullptr, *ring = nullptr;
    ZL_CHECK_CUDA(cudaMallocHost((void**)&stage, sizeof(int32_t) * (4 * B + 4 + T)));
    m->h_stage.reset(stage);
    ZL_CHECK_CUDA(cudaMallocHost((void**)&ring, sizeof(int32_t) * zl_llama::kStageSlots * 2 * B));
    m->h_ring.reset(ring);
    for (int i = 0; i < zl_llama::kStageSlots; ++i)
        ZL_CHECK_CUDA(cudaEventCreateWithFlags(&m->ring_ev[i], cudaEventDisableTiming));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    return ZL_OK;
}

// The decode-step kernel chain (captured into a graph by run_step).
// cfg.fuse: 0 = one kernel per reference operator; 1 = RMSNorm folded into the following W4 GEMM;
//           2 = additionally qkv split + RoPE + KV append folded into the qkv GEMM epilogue.
// L2 head of the successor GEMM (w4a16_gemm_v3.cu): as an exact-integer GEMM's weight stream drains, it can prefetch the
// first ZL_W4_L2_HEAD ring items of every warp of the next W4 GEMM of the decode chain, or the whole successor when it is
// at most ZL_W4_L2_WHOLE_MB.  Both default to 0 (off): on an H100 at 400 W every setting measured slower than none
// (profiles/l2_head_ab.txt).  Read once per process, so graphs capture a fixed plan.
static int l2_head_depth() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("ZL_W4_L2_HEAD");
        v = e ? atoi(e) : 0;
        if (v < 0) v = 0;
    }
    return v;
}
static size_t l2_whole_max() {
    static long v = -1;
    if (v < 0) {
        const char* e = getenv("ZL_W4_L2_WHOLE_MB");
        v = e ? atol(e) : 0;
        if (v < 0) v = 0;
    }
    return (size_t)v << 20;
}

// The launches of the decode chain, in order.  ZL_NO_PDL_MASK (experiments): bit 1 << stage launches that stage with a full
// dependency instead of a programmatic one (1 qkv GEMM, 2 attention, 4 o GEMM, 8 gate_up GEMM, 16 down GEMM, 32 final
// norm, 64 lm_head, 128 argmax / sampler).
// Single GPU, default 66 = lm_head + attention (a PDL-launched lm_head measured much slower, tools/gpu_tail.sh): on an
// H100 80GB HBM3 at 400 W, Llama-3.1-8B batch-1 decode measured 425.8 tok/s (425.6-426.2 over 5 runs) against 413.2
// (412.5-415.2) with the o GEMM also fully dependent (70), 420 with attention PDL-launched too (64), and 400-405 with
// lm_head PDL-launched (2, 0)
// (profiles/l2_head_ab.txt): an o GEMM launched early stages its ring fill while attention runs.
// Tensor parallel (exchange inside the GEMMs): 68, a PDL-launched attention kernel measured faster there.
enum Stage { kQkv, kAttn, kO, kGateUp, kDown, kFinalNorm, kLmHead, kPick };

static int stage_pdl(const zl_llama* m, Stage s) {
    static int mask = -2;
    if (mask == -2) {
        const char* e = getenv("ZL_NO_PDL_MASK");
        mask = e ? atoi(e) : -1;
    }
    const int npm = mask >= 0 ? mask : m->cfg.tp_size > 1 ? 68 : 66;
    return (npm >> s & 1) ? 0 : m->cfg.use_pdl;
}

// the successor of W4 GEMM stage s of layer l in the decode chain -- qkv -> o -> gate_up -> down -> next layer's qkv -- and
// its tensor-parallel mode given this GEMM's (the fused exchange alternates push / reduce-in; the last layer's down keeps
// the stand-alone all-reduce).  The lm_head boundary is left out.
static const W4Lin* w4_successor(zl_llama* m, int l, Stage s, int tp_mode, int* succ_tp) {
    Layer& L = m->layers[l];
    const bool last = l + 1 >= m->cfg.num_layers;
    *succ_tp = 0;
    switch (s) {
        case kQkv: *succ_tp = tp_mode ? 2 : 0; return &L.q_o;
        case kO: *succ_tp = tp_mode ? 1 : 0; return &L.q_gu;
        case kGateUp: *succ_tp = tp_mode && !last ? 2 : 0; return &L.q_down;
        case kDown: *succ_tp = tp_mode ? 1 : 0; return last ? nullptr : &m->layers[l + 1].q_qkv;
        default: return nullptr;
    }
}

// row `row` of an fp16 activation matrix of `width` columns
void* rows(const void* base, int row, int width) { return (char*)base + (size_t)row * width * 2; }

// One launch sequence of the layer GEMMs -- a decode step, one half of a dual-stream prefill chunk, or
// zl_llama_bench_gemms -- and the residual stream it updates.
struct Chain {
    enum Sink {
        kAddResidual,   // o / down add their output to the residual stream in the epilogue
        kPartial,       // o / down write partial sums to pend; the caller reduces them (dual-stream prefill)
        kAllReduce,     // tensor parallel: o / down partial sums -> one-shot all-reduce fused with the residual add
    };
    int row0 = 0, n = 0;       // rows of the activation matrices this sequence covers
    Sink sink = kAddResidual;
    bool no_pdl = false;       // full dependencies and no L2 head: the next launch is not the chain successor (dual stream)
    bool gemm_only = false;    // launch only what the GEMMs of this fuse level comprise: no stand-alone RMSNorm (fuse 0)
                               // or RoPE / KV append (fuse < 2)
    void* h = nullptr;         // current residual stream
    // Fused tensor-parallel exchange (decode-sized W4 steps): the row-parallel GEMMs (o, down but the last layer's) push
    // their fp16 partial tiles into every rank's inbox from the epilogue; the next GEMM (gate_up, next layer's qkv)
    // reduces them in rank order while it stages its activations and writes the new residual stream to ho, the other of
    // h / h2.  Producer and consumer of one exchange use the same index; the word tags in comm_dev.cuh depend on it.
    bool fused = false;
    void* ho = nullptr;
    bool pending = false;      // partial sums of the previous row-parallel GEMM are in flight to the inboxes
    int xi = 0;                // index of the next exchange of the step
    int xodd = 0;              // 2 L - 1 exchanges per step: odd -> bit 9 of tp_index

    void push(zl_w4_fused_args_t* a) {
        a->tp_mode = 2;
        a->tp_index = (xi++) | xodd;
        pending = true;
    }
    // call after a->x is taken from h
    void reduce_in(zl_w4_fused_args_t* a) {
        if (!pending) return;
        a->tp_mode = 1;
        a->tp_h_out = ho;
        a->tp_index = (xi - 1) | xodd;
        std::swap(h, ho);
        pending = false;
    }
};

// One W4 GEMM of stage s of layer l.  The caller sets a's activation, output, epilogue, RoPE and exchange fields; this adds
// the weights, the RMSNorm ln_w (fused into the GEMM or as its own kernel), the act-order gather, the PDL flag and the L2
// head of the successor.
int w4_gemm(zl_llama* m, int l, Stage s, const Chain& ch, const W4Lin& w, const void* ln_w, zl_w4_fused_args_t a) {
    const auto& c = m->cfg;
    const int route = route_of(w, ch.n);
    a.packed = route ? w.packed_i.get() : w.packed.get();
    a.variant = route ? 1 : 0;
    if (!a.packed) {
        zl_set_last_error(__FILE__, __LINE__, "no packed weight variant for this batch size");
        return ZL_ERR_STATE;
    }
    const int pdl = ch.no_pdl ? 0 : c.use_pdl;
    if (ln_w && (c.fuse == 0 || route == 4 || (w.k_perm && route != 3))) {
        // the RMSNorm runs as its own kernel (reference order, block.cpp:125,131) into the matching rows of xn: at fuse 0,
        // for the wgmma kernel, which reads x through the TMA engine, and for an act-order GEMM not gathered while staged
        void* xn = rows(m->xn.get(), ch.row0, w.K);
        if (c.fuse > 0 || !ch.gemm_only)
            RCHECK(zl_rmsnorm(a.x, ln_w, xn, ch.n, w.K, c.eps, 1.f, c.dtype, pdl, m->stream));
        a.x = xn;
        ln_w = nullptr;
    }
    if (w.k_perm && route == 3) {
        a.k_perm = w.k_perm.get();   // gathered while the integer kernel stages x
    } else if (w.k_perm) {
        // the other routes read x in tiles: permute it first (permute_input, gptq/utils.cu:322-398)
        RCHECK(zl_gather_cols_16(a.x, a.ldx, w.k_perm.get(), m->xperm.get(), ch.n, w.K, pdl, m->stream));
        a.x = m->xperm.get();
        a.ldx = w.K;
    }
    W4L2Head l2;
    if (!ch.no_pdl && route == 3 && (l2_head_depth() > 0 || l2_whole_max() > 0)) {
        int succ_tp = 0;
        const W4Lin* nx = w4_successor(m, l, s, a.tp_mode, &succ_tp);
        if (nx && route_of(*nx, ch.n) == 3)
            w4_v3_l2_head(nx->packed_i.get(), ch.n, nx->N, nx->K, succ_tp, device_sm_count(), l2_head_depth(),
                          l2_whole_max(), &l2);
    }
    a.bias = w.bias.get();
    a.M = ch.n;
    a.N = w.N;
    a.K = w.K;
    a.group_size = c.group_size;
    a.pdl = ch.no_pdl ? 0 : stage_pdl(m, s);
    a.ln_weight = ln_w;
    a.eps = c.eps;
    if (a.tp_mode) a.tp_comm = m->comm;
    return w4a16_gemm_fused_l2(&a, &l2, m->stream);
}

// int8 KV cache: the staged rotated K / V rows of ch's tokens -> codes and scales at their placement in their task's cache
// (int8_op::quant_calc_scale(x, 127, 128) + copy_to_rag_buffer2, attention.cpp:656-676)
int kv8_append(zl_llama* m, int l, const Chain& ch, int pdl) {
    const auto& c = m->cfg;
    const Layer& L = m->layers[l];
    const size_t row = (size_t)m->hkv * c.dim_head;
    const __half* ks = static_cast<const __half*>(m->kv_stage.get()) + ch.row0 * row;
    const __half* vs = static_cast<const __half*>(m->kv_stage.get()) + ((size_t)m->tok_cap + ch.row0) * row;
    return zl_kv_int8_quant_append(ks, vs, m->cur_tb + ch.row0, m->cur_pos + ch.row0, L.k_addrs.get(), L.v_addrs.get(),
                                   L.sk_addrs.get(), L.sv_addrs.get(), ch.n, m->hkv, c.dim_head, c.dtype, pdl, m->stream);
}

// int8 KV cache after a GEMM that wrote the fused qkv rows of ch: split + RoPE (zl_rope_qk_cache) into q and the staging
// rows, then quantise those into the cache -- the reference's own operator sequence (attention.cpp:636-676)
int kv8_rope_append(zl_llama* m, int l, const Chain& ch, const void* qkv, void* q, int pdl) {
    const auto& c = m->cfg;
    const int d = c.dim_head;
    const size_t row = (size_t)m->hkv * d;
    __half* ks = static_cast<__half*>(m->kv_stage.get()) + ch.row0 * row;
    __half* vs = static_cast<__half*>(m->kv_stage.get()) + ((size_t)m->tok_cap + ch.row0) * row;
    RCHECK(zl_rope_qk_cache(m->cosb.get() + (size_t)ch.row0 * d, m->sinb.get() + (size_t)ch.row0 * d, qkv, q, ks, vs, ch.n,
                            m->hq, m->hkv, d, 1, c.dtype, m->stream));
    return kv8_append(m, l, ch, pdl);
}

// qkv: RMSNorm + GEMM; at fuse >= 2 the epilogue splits q / k / v, applies RoPE and appends K / V, otherwise
// zl_qkv_rope_append does.  int8 KV cache: the epilogue appends to the staging rows instead (fuse >= 2) or
// zl_rope_qk_cache writes them (fuse < 2), and kv8_append quantises them into the cache.
int qkv_gemm(zl_llama* m, int l, Chain& ch) {
    const auto& c = m->cfg;
    const Layer& L = m->layers[l];
    const int d = c.dim_head, hqkv = (m->hq + 2 * m->hkv) * d;
    zl_w4_fused_args_t a = {};
    a.x = rows(ch.h, ch.row0, c.dim_model);
    a.ldx = c.dim_model;
    const float* cos = m->cosb.get() + (size_t)ch.row0 * d;
    const float* sin = m->sinb.get() + (size_t)ch.row0 * d;
    void* q = rows(m->q.get(), ch.row0, m->hq * d);
    const int32_t* tb = m->cur_tb + ch.row0;
    const int32_t* pos = m->cur_pos + ch.row0;
    // int8 cache at fuse >= 2 on the exact-integer route (M <= 16): the epilogue quantises K / V into the cache.  The wgmma
    // and fp16 routes, and act-order qkv, append fp16 rows to the staging rows and kv8_append quantises them.
    const bool fused_kv8 = c.kv_int8 && c.fuse >= 2 && !L.q_qkv.k_perm && route_of(L.q_qkv, ch.n) == 3;
    if (c.fuse >= 2) {
        a.epilogue = ZL_EPI_QKV_ROPE;
        a.cos = cos;
        a.sin = sin;
        a.q_out = q;
        a.token_batch = tb;
        a.placement = pos;
        a.k_addrs = L.k_addrs.get();
        a.v_addrs = L.v_addrs.get();
        a.num_heads = m->hq;
        a.num_kv_heads = m->hkv;
        a.dim_head = d;
        if (fused_kv8) {   // the exact-integer kernel quantises the rows into the cache itself
            a.kv_int8 = 1;
            a.scale_k_addrs = L.sk_addrs.get();
            a.scale_v_addrs = L.sv_addrs.get();
            a.kv8_stage = m->kv8_rows.get();
            a.kv8_counters = m->kv8_cnt.get();
        } else if (c.kv_int8) {   // staging row of token i = row row0 + i of the one "task" stage_addrs
            a.token_batch = m->d_zeros.get();
            a.placement = m->d_rowidx.get() + ch.row0;
            a.k_addrs = m->stage_addrs.get();
            a.v_addrs = m->stage_addrs.get() + 1;
        }
    } else {
        a.y = rows(m->qkv.get(), ch.row0, hqkv);
    }
    ch.reduce_in(&a);
    RCHECK(w4_gemm(m, l, kQkv, ch, L.q_qkv, L.ln_attn.get(), a));
    if (ch.gemm_only) return ZL_OK;
    const int pdl = ch.no_pdl ? 0 : c.use_pdl;
    if (fused_kv8) return ZL_OK;
    if (c.kv_int8) return c.fuse >= 2 ? kv8_append(m, l, ch, pdl) : kv8_rope_append(m, l, ch, a.y, q, pdl);
    if (c.fuse >= 2) return ZL_OK;
    return zl_qkv_rope_append(cos, sin, a.y, q, tb, pos, L.k_addrs.get(), L.v_addrs.get(), ch.n, m->hq, m->hkv, d, 1, 1,
                              m->d_lens.get(), c.dtype, pdl, m->stream);
}

// attention of B tasks x len_q query rows (tasks task0 .. task0 + B - 1) over layer l's cache: zl_decode_attention, or
// zl_decode_attention_kv8 over the int8 cache
int attention(zl_llama* m, int l, const void* q, int task0, const int8_t* mask, int max_len, void* out, int B, int len_q,
              int pdl, cudaStream_t st) {
    const auto& c = m->cfg;
    const Layer& L = m->layers[l];
    const float scale = 1.0f / sqrtf((float)c.dim_head);   // attention.cpp:89
    if (c.kv_int8)
        return zl_decode_attention_kv8(q, m->d_lens.get() + task0, L.k_addrs.get() + task0, L.v_addrs.get() + task0,
                                       L.sk_addrs.get() + task0, L.sv_addrs.get() + task0, mask, scale, max_len, out, B,
                                       len_q, m->hq, m->hkv, c.dim_head, m->attn_ws.get(), m->attn_ws_bytes, c.dtype, pdl,
                                       st);
    return zl_decode_attention(q, m->d_lens.get() + task0, L.k_addrs.get() + task0, L.v_addrs.get() + task0, mask, scale,
                               max_len, out, B, len_q, m->hq, m->hkv, c.dim_head, 1, m->attn_ws.get(), m->attn_ws_bytes,
                               c.dtype, pdl, st);
}

// gate_up: RMSNorm + GEMM + SwiGLU epilogue into act
int gate_up_gemm(zl_llama* m, int l, Chain& ch) {
    const auto& c = m->cfg;
    zl_w4_fused_args_t a = {};
    a.x = rows(ch.h, ch.row0, c.dim_model);
    a.ldx = c.dim_model;
    a.y = rows(m->act.get(), ch.row0, m->ff);
    a.epilogue = ZL_EPI_SWIGLU;
    ch.reduce_in(&a);
    return w4_gemm(m, l, kGateUp, ch, m->layers[l].q_gu, m->layers[l].ln_ff.get(), a);
}

// o (input ao) and down (input act): row-parallel under tensor parallelism, their output goes to ch.sink
int row_parallel_gemm(zl_llama* m, int l, Stage s, Chain& ch) {
    const auto& c = m->cfg;
    const W4Lin& w = s == kO ? m->layers[l].q_o : m->layers[l].q_down;
    zl_w4_fused_args_t a = {};
    a.x = rows(s == kO ? m->ao.get() : m->act.get(), ch.row0, w.K);
    a.ldx = w.K;
    // the last layer's down keeps the stand-alone all-reduce: the final norm is not a GEMM
    const bool push = ch.fused && (s == kO || l + 1 < c.num_layers);
    if (push) {
        ch.push(&a);
    } else if (ch.sink == Chain::kAddResidual) {
        a.residual = a.y = rows(ch.h, ch.row0, c.dim_model);
        a.epilogue = ZL_EPI_RESIDUAL;
    } else {
        a.y = rows(m->pend.get(), ch.row0, c.dim_model);
    }
    RCHECK(w4_gemm(m, l, s, ch, w, nullptr, a));
    if (push || ch.sink != Chain::kAllReduce) return ZL_OK;
    return zl_allreduce_one_shot(m->comm, a.y, ch.h, ch.h, (size_t)ch.n * c.dim_model, c.dtype, c.tp_int8,
                                 ch.no_pdl ? 0 : c.use_pdl, m->stream);
}
int o_gemm(zl_llama* m, int l, Chain& ch) { return row_parallel_gemm(m, l, kO, ch); }
int down_gemm(zl_llama* m, int l, Chain& ch) { return row_parallel_gemm(m, l, kDown, ch); }

// One non-W4 Linear of the decode chain: dense (NormalLinear), or W8A8 = activation quant + fused 8-bit GEMM
// (Int8Linear::forward / Fp8Linear::forward in two launches instead of three).
int dense_or_w8(zl_llama* m, const void* x, const DenseLin& L, void* y, int B, int pdl) {
    const auto& c = m->cfg;
    cudaStream_t st = m->stream;
    if (!L.w8) return zl_dense_gemm_skinny(x, L.K, L.w.get(), L.bias.get(), y, B, L.N, L.K, c.dtype, c.dtype, pdl, st);
    if (L.w8_kind == ZL_W8_INT8) {
        RCHECK(zl_int8_quant_per_token(x, L.K, m->xq.get(), m->xs.get(), B, L.K, c.dtype, pdl, st));
        return zl_w8a8_gemm(m->xq.get(), m->xs.get(), L.w8.get(), L.w_scale.get(), c.dtype, L.bias.get(), y, B, L.N, L.K,
                            ZL_W8_INT8, c.dtype, pdl, st);
    }
    if (L.w8_kind == kW8Block) {   // Fp8Block::forward: per_token_cast_to_fp8 + the block-scaled GEMM
        const int ld = (B + 3) / 4 * 4;
        RCHECK(zl_fp8_quant_per_token_group(x, L.K, m->xq.get(), m->xs.get(), ld, B, L.K, c.dtype, pdl, st));
        return zl_fp8_block_gemm(m->xq.get(), m->xs.get(), ld, L.w8.get(), static_cast<const float*>(L.w_scale.get()), y,
                                 B, L.N, L.K, c.dtype, pdl, st);
    }
    RCHECK(zl_fp8_quant_per_tensor(x, m->xq.get(), m->xs.get(), (size_t)B * L.K, c.dtype, pdl, st));
    return zl_w8a8_gemm(m->xq.get(), m->xs.get(), L.w8.get(), L.w_scale.get(), ZL_F32, L.bias.get(), y, B, L.N, L.K,
                        ZL_W8_FP8_ROWS, c.dtype, pdl, st);
}

// pf != nullptr: a list of segments -- rows of one task at consecutive positions -- instead of one token per task.  Their
// tokens, positions and token -> task map are staged in d_pf_tokens / d_pf_pos / d_tb.
//   prefill chunk (joined = false): ONE segment (task, pos0, n), attended with the masked decode kernel; last = run the
//                                   final norm + lm_head + pick on its last row
//   joined step (joined = true):    nseg segments of distinct tasks (d_join), attended with zl_varlen_attention; the last
//                                   rows of the n_emit emitting segments feed the head
struct Segments {
    int task = 0, pos0 = 0, n = 0;   // n: rows of the whole launch sequence
    bool last = false;
    bool joined = false;
    int nseg = 1, n_emit = 0, max_keys = 0;
};

// ------------------------------------------------------------------------------------------------------------------
// Dual-stream chunked prefill of a W4 model (EncoderLayer::impl::dual_stream_encode, src/nn/block/block.cpp:205-441):
// the chunk's tokens are split in two halves that walk the layers as a 2-stage pipeline -- while the reduce stream
// combines half A's row-parallel partial sums (NVLink all-reduce fused with the residual add; a plain residual add when
// tp_size == 1), the compute stream already runs half B's GEMMs / attention.  The reference creates its second stream
// and 2*num_split events on every forward (block.cpp:220-224, 260-267); here they live in the model object.
//   compute: S1(h0) S1(h1) S3(h0) S3(h1) | next layer ...      S1 = qkv(+RoPE, KV append) -> attention -> o GEMM
//   reduce :        R1(h0) R1(h1) R2(h0) R2(h1)                S3 = gate_up (SwiGLU) -> down GEMM ; R = reduce + residual
// ------------------------------------------------------------------------------------------------------------------
int ensure_dual_resources(zl_llama* m) {
    if (m->reduce_stream) return ZL_OK;
    ZL_CHECK_CUDA(cudaStreamCreateWithFlags(&m->reduce_stream, cudaStreamNonBlocking));
    for (int h = 0; h < 2; ++h)
        for (cudaEvent_t* e : {&m->ev_o[h], &m->ev_r1[h], &m->ev_dn[h], &m->ev_r2[h]})
            ZL_CHECK_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    return ZL_OK;
}

static bool prefill_dual_enabled(const zl_llama* m, int n) {
    // ZL_PREFILL_DUAL: 0 never, 1 always (on one GPU the "reduce" is the residual add: exercises the pipeline),
    // 2 (default) = when tensor parallel.  Read per call: prefill is not a latency-critical path.
    const char* e = getenv("ZL_PREFILL_DUAL");
    const int force = e ? atoi(e) : 2;
    const auto& c = m->cfg;
    if (!(c.quant_type == 5 || c.quant_type == 6) || c.fuse < 1 || n < 16) return false;
    return force == 1 || (force == 2 && c.tp_size > 1);
}

int prefill_layers_dual(zl_llama* m, const Segments& pf) {
    const auto& c = m->cfg;
    RCHECK(ensure_dual_resources(m));
    const int D = c.dim_model, d = c.dim_head, dt = c.dtype;
    const bool tp = c.tp_size > 1;
    cudaStream_t cs = m->stream, rs = m->reduce_stream;
    const int n0 = (pf.n / 2 + 7) / 8 * 8 < pf.n ? (pf.n / 2 + 7) / 8 * 8 : pf.n / 2;   // rows of half 0
    const int len_buf = pf.pos0 + pf.n;
    Chain half[2];
    for (int h = 0; h < 2; ++h) {
        half[h].row0 = h ? n0 : 0;
        half[h].n = h ? pf.n - n0 : n0;
        half[h].sink = Chain::kPartial;
        half[h].no_pdl = true;
        half[h].h = m->h.get();
    }
    auto reduce = [&](const Chain& ch) -> int {   // h rows: h += sum over ranks of pend
        void* hp = rows(m->h.get(), ch.row0, D);
        void* pp = rows(m->pend.get(), ch.row0, D);
        if (tp) return zl_allreduce_one_shot(m->comm, pp, hp, hp, (size_t)ch.n * D, dt, c.tp_int8, 0, rs);
        return zl_element_add_scale(hp, pp, hp, (size_t)ch.n * D, 1.0f, dt, rs);
    };
    for (int l = 0; l < c.num_layers; ++l) {
        for (int h = 0; h < 2; ++h) {   // S1
            if (l > 0) ZL_CHECK_CUDA(cudaStreamWaitEvent(cs, m->ev_r2[h], 0));
            const int r0 = half[h].row0;
            RCHECK(qkv_gemm(m, l, half[h]));
            // causal rows r0.. of the chunk's mask; keys of BOTH halves are visible as far as the mask allows, so half 1
            // needs half 0's K/V rows, which the same stream appended just before
            RCHECK(attention(m, l, rows(m->q.get(), r0, m->hq * d), pf.task, m->d_mask.get() + (size_t)r0 * len_buf, len_buf,
                             rows(m->ao.get(), r0, m->hq * d), 1, half[h].n, 0, cs));
            RCHECK(o_gemm(m, l, half[h]));
            ZL_CHECK_CUDA(cudaEventRecord(m->ev_o[h], cs));
            ZL_CHECK_CUDA(cudaStreamWaitEvent(rs, m->ev_o[h], 0));   // R1
            RCHECK(reduce(half[h]));
            ZL_CHECK_CUDA(cudaEventRecord(m->ev_r1[h], rs));
        }
        for (int h = 0; h < 2; ++h) {   // S3
            ZL_CHECK_CUDA(cudaStreamWaitEvent(cs, m->ev_r1[h], 0));
            RCHECK(gate_up_gemm(m, l, half[h]));
            RCHECK(down_gemm(m, l, half[h]));
            ZL_CHECK_CUDA(cudaEventRecord(m->ev_dn[h], cs));
            ZL_CHECK_CUDA(cudaStreamWaitEvent(rs, m->ev_dn[h], 0));   // R2
            RCHECK(reduce(half[h]));
            ZL_CHECK_CUDA(cudaEventRecord(m->ev_r2[h], rs));
        }
    }
    for (int h = 0; h < 2; ++h) ZL_CHECK_CUDA(cudaStreamWaitEvent(cs, m->ev_r2[h], 0));
    return ZL_OK;
}

int enqueue_step(zl_llama* m, int n_tasks, int len_bucket, const Segments* pf = nullptr, bool sampler = false) {
    const auto& c = m->cfg;
    const int B = pf ? pf->n : n_tasks;   // rows (tokens) of every activation matrix in this launch sequence
    const int D = c.dim_model, d = c.dim_head, dt = c.dtype, pdl = c.use_pdl;
    cudaStream_t st = m->stream;
    const bool w4 = c.quant_type == 5 || c.quant_type == 6;
    const bool tp = c.tp_size > 1;
    const bool joined = pf && pf->joined;
    if (tp && !m->comm) {
        zl_set_last_error(__FILE__, __LINE__, "tp_size > 1 but zl_llama_set_comm was not called");
        return ZL_ERR_STATE;
    }
    // joined steps: d_join = segments (nseg x 4) | emitting rows | their tasks | their positions (max_batch each)
    const int32_t* j_seg = joined ? m->d_join.get() : nullptr;
    const int32_t* j_rows = joined ? j_seg + 4 * c.max_batch : nullptr;
    const int32_t* j_task = joined ? j_rows + c.max_batch : nullptr;
    const int32_t* j_pos = joined ? j_task + c.max_batch : nullptr;

    // (a joined step's positions and token -> task map were staged by zl_llama_step_joined with its tokens)
    if (pf && !joined) {
        k_prefill_setup<<<8, 256, 0, st>>>(m->d_pf_pos.get(), m->d_tb.get(), m->d_lens.get(), m->d_mask.get(), pf->task,
                                           pf->pos0, pf->n);
        ZL_CHECK_LAUNCH();
    } else if (!pf) {
        ZL_CHECK_CUDA(launch(k_lens_from_pos, dim3(cdiv(B, 64)), dim3(64), 0, st, false, (const int32_t*)m->d_pos.get(),
                             m->d_lens.get(), B, g_w4_trace));
    }
    m->cur_tb = pf ? m->d_tb.get() : m->d_iota.get();
    m->cur_pos = pf ? m->d_pf_pos.get() : m->d_pos.get();
    m->cur_tokens = pf ? m->d_pf_tokens.get() : m->d_tokens.get();
    RCHECK(zl_rope_cos_sin(m->cur_pos, m->cosb.get(), m->sinb.get(), B, d, c.rope_theta, c.rope_llama3_factor,
                           c.rope_low_freq_factor, c.rope_high_freq_factor, c.rope_orig_ctx, 1, st));
    RCHECK(zl_embedding(m->cur_tokens, m->emb.get(), m->h.get(), B, D, c.vocab_size, dt, 0, st));
    const bool dual = pf && !joined && prefill_dual_enabled(m, pf->n);
    if (dual) RCHECK(prefill_layers_dual(m, *pf));
    Chain ch;
    ch.n = B;
    ch.sink = tp ? Chain::kAllReduce : Chain::kAddResidual;
    ch.h = m->h.get();
    ch.ho = m->h2.get();
    // Tensor parallel, decode-sized launches of a W4 model: the exchange rides inside the GEMMs (Chain).  ZL_TP_UNFUSED=1
    // keeps the separate exchange kernels everywhere (A/B).
    ch.fused = tp && w4 && !pf && c.fuse >= 1 && !c.tp_int8 && dt == ZL_F16 && !getenv("ZL_TP_UNFUSED") &&
               (size_t)B * D * 2 <= zl_comm_slot_bytes(m->comm) && 2 * c.num_layers <= 512;
    if (ch.fused) {
        const Layer& L0 = m->layers[0];
        for (const W4Lin* w : {&L0.q_qkv, &L0.q_o, &L0.q_gu, &L0.q_down})
            if (route_of(*w, B) != 3) ch.fused = false;
    }
    if (ch.fused) RCHECK(zl_comm_ll_begin_step(m->comm, st));   // the word tags of this step's exchanges
    ch.xodd = ((2 * c.num_layers - 1) & 1) << 9;
    for (int l = 0; l < (dual ? 0 : c.num_layers); ++l) {
        Layer& L = m->layers[l];
        if (w4) {
            RCHECK(qkv_gemm(m, l, ch));
        } else {
            // residual of the previous layer's FFN is folded into this norm (block.cpp:139-141 + 131)
            RCHECK(zl_add_rmsnorm(m->h.get(), l == 0 ? nullptr : m->pend.get(), L.ln_attn.get(), m->h.get(), m->xn.get(),
                                  B, D, c.eps, 1.f, 0, dt, pdl, st));
            RCHECK(dense_or_w8(m, m->xn.get(), L.d_qkv, m->qkv.get(), B, pdl));
            if (c.kv_int8) {
                RCHECK(kv8_rope_append(m, l, ch, m->qkv.get(), m->q.get(), pdl));
            } else {
                RCHECK(zl_qkv_rope_append(m->cosb.get(), m->sinb.get(), m->qkv.get(), m->q.get(), m->cur_tb, m->cur_pos,
                                          L.k_addrs.get(), L.v_addrs.get(), B, m->hq, m->hkv, d, 1, 1, m->d_lens.get(), dt,
                                          pdl, st));
            }
        }
        if (joined) {
            // every segment causally over its own task's cache, one launch (attention.cpp:924-961)
            RCHECK(zl_varlen_attention(m->q.get(), j_seg, pf->nseg, B, L.k_addrs.get(), L.v_addrs.get(),
                                       1.0f / sqrtf((float)d), pf->max_keys, m->ao.get(), m->hq, m->hkv, d, m->attn_ws.get(),
                                       m->attn_ws_bytes, dt, pdl, st));
        } else if (pf) {
            // one task, len_q = chunk, causal int8 mask (Attention::dynamic_batch_forward with len_q > 1, attention.cpp:846-964)
            RCHECK(attention(m, l, m->q.get(), pf->task, m->d_mask.get(), pf->pos0 + pf->n, m->ao.get(), 1, pf->n, pdl, st));
        } else {
            RCHECK(attention(m, l, m->q.get(), 0, nullptr, len_bucket, m->ao.get(), B, 1, stage_pdl(m, kAttn), st));
        }
        if (w4) {
            RCHECK(o_gemm(m, l, ch));
            RCHECK(gate_up_gemm(m, l, ch));
            RCHECK(down_gemm(m, l, ch));
        } else {
            RCHECK(dense_or_w8(m, m->ao.get(), L.d_o, m->pend.get(), B, pdl));
            if (tp)
                RCHECK(zl_allreduce_one_shot(m->comm, m->pend.get(), nullptr, m->pend.get(), (size_t)B * D, dt, c.tp_int8,
                                             pdl, st));
            RCHECK(zl_add_rmsnorm(m->h.get(), m->pend.get(), L.ln_ff.get(), m->h.get(), m->xn.get(), B, D, c.eps, 1.f, 0,
                                  dt, pdl, st));
            RCHECK(dense_or_w8(m, m->xn.get(), L.d_gu, m->gu.get(), B, pdl));
            RCHECK(zl_gate_mul(m->gu.get(), 2 * m->ff, (char*)m->gu.get() + (size_t)m->ff * 2, 2 * m->ff, m->act.get(),
                               m->ff, B, m->ff, 0, dt, st));
            RCHECK(dense_or_w8(m, m->act.get(), L.d_down, m->pend.get(), B, pdl));
            if (tp)
                RCHECK(zl_allreduce_one_shot(m->comm, m->pend.get(), nullptr, m->pend.get(), (size_t)B * D, dt, c.tp_int8,
                                             pdl, st));
        }
    }
    const void* head_x = m->xn.get();   // rows that reach lm_head
    if (joined) {
        if (pf->n_emit == 0) return ZL_OK;
        // the final norm is row-wise: norm every row, then gather the emitting segments' last rows into rows
        // 0 .. n_emit - 1 of pend (free after the norm), so that only they reach lm_head
        if (w4)
            RCHECK(zl_rmsnorm(m->h.get(), m->ln_f.get(), m->xn.get(), B, D, c.eps, 1.f, dt, pdl, st));
        else
            RCHECK(zl_add_rmsnorm(m->h.get(), m->pend.get(), m->ln_f.get(), m->h.get(), m->xn.get(), B, D, c.eps, 1.f, 0,
                                  dt, pdl, st));
        k_gather_rows<<<pf->n_emit, 256, 0, st>>>(static_cast<const uint16_t*>(m->xn.get()), j_rows,
                                                 static_cast<uint16_t*>(m->pend.get()), D);
        ZL_CHECK_LAUNCH();
        head_x = m->pend.get();
    } else if (pf) {
        if (!pf->last) return ZL_OK;
        // only the last prompt position feeds the head: move it to row 0 semantics by pointing at its row
        void* hl = rows(m->h.get(), pf->n - 1, D);
        if (w4) {
            RCHECK(zl_rmsnorm(hl, m->ln_f.get(), m->xn.get(), 1, D, c.eps, 1.f, dt, pdl, st));
        } else {
            RCHECK(zl_add_rmsnorm(hl, rows(m->pend.get(), pf->n - 1, D), m->ln_f.get(), hl, m->xn.get(), 1, D, c.eps, 1.f,
                                  0, dt, pdl, st));
        }
    } else if (w4) {
        RCHECK(zl_rmsnorm(ch.h, m->ln_f.get(), m->xn.get(), B, D, c.eps, 1.f, dt, stage_pdl(m, kFinalNorm), st));
    } else {
        RCHECK(zl_add_rmsnorm(m->h.get(), m->pend.get(), m->ln_f.get(), m->h.get(), m->xn.get(), B, D, c.eps, 1.f, 0, dt,
                              stage_pdl(m, kFinalNorm), st));
    }
    const int HB = joined ? pf->n_emit : pf ? 1 : B;   // rows that reach lm_head
    // vocab-parallel lm_head (embedding.cu:353-392): each rank owns vshard rows
    RCHECK(zl_dense_gemm_skinny(head_x, D, m->lm_head, nullptr, m->logits.get(), HB, m->vshard, D, dt, ZL_F32,
                                stage_pdl(m, kLmHead), st));
    if (sampler) {
        // one row per task at decode (row b = task b, counter = its input position); prefill: the task's last prompt
        // position; joined: each emitting segment's task and last position.  set_sampling keeps this off under tensor
        // parallelism.
        const int32_t* row_task = joined ? j_task : pf ? m->d_iota.get() + pf->task : m->d_iota.get();
        const int32_t* counter = joined ? j_pos : pf ? m->d_pf_pos.get() + (pf->n - 1) : m->d_pos.get();
        RCHECK(zl_sample(m->logits.get(), HB, m->vshard, m->d_sparams.get(), row_task, counter, m->d_hist.get(), m->hwords,
                         m->d_next.get(), nullptr, 0, stage_pdl(m, kPick), st));
    } else if (!tp) {
        RCHECK(zl_argmax(m->logits.get(), m->d_next.get(), HB, m->vshard, m->argmax_ws.get(), zl_argmax_workspace_bytes(HB),
                         stage_pdl(m, kPick), st));
    } else {
        // instead of all-gathering (B, V) logits, exchange one {value, index} candidate per token
        const int stride = ((HB * 8 + 15) / 16) * 2;   // int2 records per rank slot (16-byte multiple)
        RCHECK(zl_argmax_candidates(m->logits.get(), m->cand.get(), HB, m->vshard, c.tp_rank * m->vshard,
                                    m->argmax_ws.get(), zl_argmax_workspace_bytes(HB), pdl, st));
        RCHECK(zl_allgather_small(m->comm, m->cand.get(), m->cand_all.get(), (size_t)stride * 8, pdl, st));
        RCHECK(zl_argmax_merge(m->cand_all.get(), m->d_next.get(), HB, c.tp_size, stride, pdl, st));
    }
    return ZL_OK;
}

// attention split counts are baked into the graph: one graph per (batch, length bucket)
int len_bucket_of(const zl_llama* m, int max_len) {
    int b = 256;
    while (b < max_len) b <<= 1;
    return b < m->cfg.max_seq ? b : (m->cfg.max_seq > 256 ? m->cfg.max_seq : 256);
}

bool sampler_on(const zl_llama* m, int first, int n) {
    for (int t = first; t < first + n; ++t)
        if (m->samp_on[t]) return true;
    return false;
}

int run_step(zl_llama* m, int B) {
    const int bucket = len_bucket_of(m, m->cur_max_len);
    const bool sampler = sampler_on(m, 0, B);
    if (!m->cfg.use_graph) return enqueue_step(m, B, bucket, nullptr, sampler);
    // parameter changes need no re-capture (they live on the device), only switching the sampler on or off does
    const long long key = ((long long)B << 33) | ((long long)sampler << 32) | (unsigned)bucket;
    auto it = m->graphs.find(key);
    if (it == m->graphs.end()) {
        cudaGraph_t graph = nullptr;
        ZL_CHECK_CUDA(cudaStreamBeginCapture(m->stream, cudaStreamCaptureModeThreadLocal));
        int rc = enqueue_step(m, B, bucket, nullptr, sampler);
        cudaError_t ce = cudaStreamEndCapture(m->stream, &graph);
        if (rc != ZL_OK) {
            if (graph) cudaGraphDestroy(graph);
            return rc;
        }
        ZL_CHECK_CUDA(ce);
        cudaGraphExec_t exec = nullptr;
        ZL_CHECK_CUDA(cudaGraphInstantiate(&exec, graph, 0));
        size_t n_nodes = 0;
        cudaGraphGetNodes(graph, nullptr, &n_nodes);
        m->kernels_per_step = (int)n_nodes;
        cudaGraphDestroy(graph);
        it = m->graphs.emplace(key, exec).first;
    }
    ZL_CHECK_CUDA(cudaGraphLaunch(it->second, m->stream));
    return ZL_OK;
}

}  // namespace

extern "C" int zl_llama_create(const zl_llama_config_t* cfg, zl_llama_t** out) {
    ZL_CHECK_ARG(cfg && out);
    ZL_CHECK_ARG(cfg->num_layers > 0 && cfg->dim_model > 0 && cfg->num_heads > 0 && cfg->num_kv_heads > 0);
    ZL_CHECK_ARG(cfg->dim_head > 0 && cfg->dim_ff > 0 && cfg->vocab_size > 0 && cfg->max_batch > 0 &&
                 cfg->max_seq > 0);
    // QuantType 8 (GPTQ_Marlin, linear.cpp:1247-1451) loads the same GPTQ checkpoint as 5 and requires the symmetric
    // u4b8 form (linear.cpp:1418-1435): it is served by the same kernels with sym = 1 (no Marlin repack needed).
    zl_llama_config_t norm_cfg = *cfg;
    if (norm_cfg.quant_type == 8) {
        norm_cfg.quant_type = 5;
        norm_cfg.sym = 1;
    }
    cfg = &norm_cfg;
    ZL_CHECK_SUPPORTED(cfg->quant_type == 0 || cfg->quant_type == 2 || cfg->quant_type == 5 || cfg->quant_type == 6 ||
                       cfg->quant_type == 7 || cfg->quant_type == 10);
    // Fp8Block (QuantType 10): single rank, no bias (Fp8Block::set_has_bias throws)
    ZL_CHECK_SUPPORTED(cfg->quant_type != 10 || (cfg->tp_size == 1 && !cfg->qkv_bias));
    // ... and 128-wide scale blocks: every K is a multiple of 128, and so is every part of the fused q/k/v and gate/up
    ZL_CHECK_SUPPORTED(cfg->quant_type != 10 ||
                       (cfg->dim_model % 128 == 0 && (cfg->num_heads * cfg->dim_head) % 128 == 0 &&
                        (cfg->num_kv_heads * cfg->dim_head) % 128 == 0 && cfg->dim_ff % 128 == 0));
    ZL_CHECK_SUPPORTED(!(cfg->quant_type == 5 || cfg->quant_type == 6) || cfg->dtype == ZL_F16);
    ZL_CHECK_SUPPORTED(!(cfg->quant_type == 2 || cfg->quant_type == 7) || cfg->tp_size == 1);   // "A must be half" q_gemm_k_major.cu:989
    ZL_CHECK_SUPPORTED(cfg->dtype == ZL_F16 || cfg->dtype == ZL_BF16);
    ZL_CHECK_SUPPORTED(cfg->tp_size >= 1 && cfg->tp_rank >= 0 && cfg->tp_rank < cfg->tp_size);
    ZL_CHECK_SUPPORTED(cfg->num_heads % cfg->tp_size == 0 && cfg->num_kv_heads % cfg->tp_size == 0 &&
                       cfg->dim_ff % cfg->tp_size == 0 && cfg->vocab_size % cfg->tp_size == 0);
    ZL_CHECK_SUPPORTED(!(cfg->quant_type == 5 || cfg->quant_type == 6) || cfg->group_size == zl::kW4GroupK);
    ZL_CHECK_ARG(cfg->fuse >= 0 && cfg->fuse <= 3);
    ZL_CHECK_ARG(cfg->prefill_chunk >= 0 && cfg->prefill_chunk <= 2048);
    ZL_CHECK_SUPPORTED(cfg->fuse < 2 || cfg->dim_head % 32 == 0);
    ZL_CHECK_ARG(cfg->kv_int8 == 0 || cfg->kv_int8 == 1);
    if (cfg->kv_int8) {
        // zl_decode_attention_kv8 takes fp16 q, d = 64 or 128, and at most 64 key splits of 1024 keys
        if (cfg->dtype != ZL_F16 || (cfg->dim_head != 64 && cfg->dim_head != 128) || cfg->max_seq > 65536)
            return fail_state(__LINE__, "kv_int8 needs dtype fp16, dim_head 64 or 128 and max_seq <= 65536",
                              ZL_ERR_UNSUPPORTED);
    }
    RCHECK(zl_prepare());
    zl_llama* m = new zl_llama();
    m->cfg = *cfg;
    m->hq = cfg->num_heads / cfg->tp_size;
    m->hkv = cfg->num_kv_heads / cfg->tp_size;
    m->ff = cfg->dim_ff / cfg->tp_size;
    m->vshard = cfg->vocab_size / cfg->tp_size;
    m->layers.resize(cfg->num_layers);
    if (cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete m;
        zl_set_last_error(__FILE__, __LINE__, "cudaStreamCreate failed (no CUDA device? there is no CPU fallback)");
        return ZL_ERR_CUDA;
    }
    *out = m;
    return ZL_OK;
}

extern "C" int zl_llama_set_comm(zl_llama_t* m, zl_comm_t* comm) {
    ZL_CHECK_ARG(m && comm);
    ZL_CHECK_ARG(zl_comm_world_size(comm) == m->cfg.tp_size && zl_comm_rank(comm) == m->cfg.tp_rank);
    m->comm = comm;
    return ZL_OK;
}

extern "C" void zl_llama_destroy(zl_llama_t* m) {
    if (!m) return;
    cudaStreamSynchronize(m->stream);
    if (m->reduce_stream) cudaStreamSynchronize(m->reduce_stream);
    for (auto& g : m->graphs) cudaGraphExecDestroy(g.second);
    for (int h = 0; h < 2; ++h)
        for (cudaEvent_t e : {m->ev_o[h], m->ev_r1[h], m->ev_dn[h], m->ev_r2[h]})
            if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : m->ring_ev)
        if (e) cudaEventDestroy(e);
    if (m->reduce_stream) cudaStreamDestroy(m->reduce_stream);
    cudaStreamDestroy(m->stream);
    delete m;   // the members free their device and pinned buffers
}

extern "C" int zl_llama_load_tensor(zl_llama_t* m, const char* name, const void* data_host, int rows, int cols,
                                    int elem_bytes) {
    ZL_CHECK_ARG(m && name && data_host && rows > 0 && cols > 0 && elem_bytes > 0);
    if (m->finalized) {
        zl_set_last_error(__FILE__, __LINE__, "model already finalized");
        return ZL_ERR_STATE;
    }
    Staged s;
    s.rows = rows;
    s.cols = cols;
    s.elem = elem_bytes;
    const size_t bytes = (size_t)rows * cols * elem_bytes;
    RCHECK(dmalloc(&s.ptr, bytes));
    ZL_CHECK_CUDA(cudaMemcpyAsync(s.ptr.get(), data_host, bytes, cudaMemcpyHostToDevice, m->stream));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    m->staged[name] = std::move(s);
    return ZL_OK;
}

extern "C" int zl_llama_finalize(zl_llama_t* m) {
    ZL_CHECK_ARG(m);
    if (m->finalized) return ZL_OK;
    for (int l = 0; l < m->cfg.num_layers; ++l)
        if (!m->layers[l].ln_attn) RCHECK(finalize_layer(m, l));
    RCHECK(finalize_globals(m));
    RCHECK(alloc_runtime(m));
    m->finalized = true;
    return ZL_OK;
}

namespace {
int stage_random(zl_llama* m, const std::string& name, int rows, int cols, int elem, int kind, float lo, float hi,
                 uint64_t seed) {
    Staged s;
    s.rows = rows;
    s.cols = cols;
    s.elem = elem;
    const size_t n = (size_t)rows * cols;
    RCHECK(dmalloc(&s.ptr, n * elem));
    uint64_t h = seed;
    for (char ch : name) h = h * 1099511628211ull + (unsigned char)ch;
    if (kind == 0)
        RCHECK(zl_fill_random_u32((uint32_t*)s.ptr.get(), n, h, m->stream));
    else if (kind == 1)
        RCHECK(zl_fill_const_u32((uint32_t*)s.ptr.get(), n, 0x77777777u, m->stream));
    else
        RCHECK(zl_fill_uniform(s.ptr.get(), n, lo, hi, h, m->cfg.dtype, m->stream));
    m->staged[name] = std::move(s);
    return ZL_OK;
}

int stage_random_linear(zl_llama* m, const std::string& prefix, int K, int N, uint64_t seed) {
    const auto& c = m->cfg;
    if (c.quant_type == 5) {
        const int G = K / c.group_size;
        RCHECK(stage_random(m, prefix + ".qweight", K / 8, N, 4, 0, 0, 0, seed));
        if (c.sym) {
            const size_t words = (size_t)(K / 8) * N;
            k_recentre_nibbles<<<(unsigned)((words + 255) / 256), 256, 0, m->stream>>>(
                static_cast<uint32_t*>(m->staged[prefix + ".qweight"].ptr.get()), words);
            ZL_CHECK_LAUNCH();
        }
        RCHECK(stage_random(m, prefix + ".qzeros", G, N / 8, 4, c.sym ? 1 : 0, 0, 0, seed));
        RCHECK(stage_random(m, prefix + ".scales", G, N, 2, 2, 0.002f, 0.006f, seed));   // SURVEY 8d config 3
    } else if (c.quant_type == 6) {
        const int G = K / c.group_size;
        RCHECK(stage_random(m, prefix + ".qweight", K, N / 8, 4, 0, 0, 0, seed));
        RCHECK(stage_random(m, prefix + ".qzeros", G, N / 8, 4, 0, 0, 0, seed));
        RCHECK(stage_random(m, prefix + ".scales", G, N, 2, 2, 0.002f, 0.006f, seed));
    } else if (c.quant_type == 7) {
        // random e4m3 codes with the exponent MSB cleared (|w| < 2, no NaN encodings) and a per-tensor scale
        RCHECK(stage_random(m, prefix + ".weight", N, K / 4, 4, 0, 0, 0, seed));
        Staged& w = m->staged[prefix + ".weight"];
        const size_t words = (size_t)N * K / 4;
        k_and_u32<<<(unsigned)((words + 255) / 256), 256, 0, m->stream>>>(static_cast<uint32_t*>(w.ptr.get()), words, 0xBFBFBFBFu);
        ZL_CHECK_LAUNCH();
        w.cols = K;
        w.elem = 1;
        Staged sc;
        sc.rows = sc.cols = 1;
        sc.elem = 4;
        RCHECK(dmalloc(&sc.ptr, 4));
        k_set_f32<<<1, 1, 0, m->stream>>>(static_cast<float*>(sc.ptr.get()), 0.03f);
        ZL_CHECK_LAUNCH();
        m->staged[prefix + ".weight_scale"] = std::move(sc);
    } else if (c.quant_type == 10) {
        // e4m3 codes as for type 7, and one f32 scale per 128x128 block drawn log-uniformly over 0.0075 .. 0.12 (16x)
        // so that a scale applied to the wrong block shows
        RCHECK(stage_random(m, prefix + ".weight", N, K / 4, 4, 0, 0, 0, seed));
        Staged& w = m->staged[prefix + ".weight"];
        const size_t words = (size_t)N * K / 4;
        k_and_u32<<<(unsigned)((words + 255) / 256), 256, 0, m->stream>>>(static_cast<uint32_t*>(w.ptr.get()), words, 0xBFBFBFBFu);
        ZL_CHECK_LAUNCH();
        w.cols = K;
        w.elem = 1;
        const int nb = (N + 127) / 128, kb = K / 128;
        RCHECK(stage_random(m, prefix + ".weight_scale_inv", nb, kb, 4, 0, 0, 0, seed));
        Staged& sc = m->staged[prefix + ".weight_scale_inv"];
        k_u32_to_log_uniform<<<cdiv(nb * kb, 256), 256, 0, m->stream>>>(static_cast<uint32_t*>(sc.ptr.get()), nb * kb,
                                                                        0.0075f, 0.12f);
        ZL_CHECK_LAUNCH();
    } else {
        RCHECK(stage_random(m, prefix + ".weight", N, K, 2, 2, -0.035f, 0.035f, seed));   // ~ randn*0.02
    }
    return ZL_OK;
}
}  // namespace

extern "C" int zl_llama_init_synthetic(zl_llama_t* m, uint64_t seed) {
    ZL_CHECK_ARG(m);
    if (m->finalized) {
        zl_set_last_error(__FILE__, __LINE__, "model already finalized");
        return ZL_ERR_STATE;
    }
    const auto& c = m->cfg;
    const int D = c.dim_model, d = c.dim_head;
    for (int l = 0; l < c.num_layers; ++l) {
        const std::string p = "layers." + std::to_string(l) + ".";
        RCHECK(stage_random(m, p + "ln_attn.weight", 1, D, 2, 2, 0.9f, 1.1f, seed));
        RCHECK(stage_random(m, p + "ln_ff.weight", 1, D, 2, 2, 0.9f, 1.1f, seed));
        RCHECK(stage_random_linear(m, p + "attn.project_q", D, m->hq * d, seed));
        RCHECK(stage_random_linear(m, p + "attn.project_k", D, m->hkv * d, seed));
        RCHECK(stage_random_linear(m, p + "attn.project_v", D, m->hkv * d, seed));
        if (c.qkv_bias) {
            RCHECK(stage_random(m, p + "attn.project_q.bias", 1, m->hq * d, 2, 2, -0.03f, 0.03f, seed));
            RCHECK(stage_random(m, p + "attn.project_k.bias", 1, m->hkv * d, 2, 2, -0.03f, 0.03f, seed));
            RCHECK(stage_random(m, p + "attn.project_v.bias", 1, m->hkv * d, 2, 2, -0.03f, 0.03f, seed));
        }
        RCHECK(stage_random_linear(m, p + "attn.attn_out", m->hq * d, D, seed));
        RCHECK(stage_random_linear(m, p + "ff.w_in", D, m->ff, seed));
        RCHECK(stage_random_linear(m, p + "ff.w_gated", D, m->ff, seed));
        RCHECK(stage_random_linear(m, p + "ff.w_out", m->ff, D, seed));
        RCHECK(finalize_layer(m, l));   // bound the staging memory to one layer
    }
    RCHECK(stage_random(m, "token_embedding.weight", c.vocab_size, D, 2, 2, -0.035f, 0.035f, seed));
    RCHECK(stage_random(m, "output_layernorm.weight", 1, D, 2, 2, 0.9f, 1.1f, seed));
    RCHECK(stage_random(m, "lm_head.weight", m->vshard, D, 2, 2, -0.035f, 0.035f, seed + 7919 * c.tp_rank));
    return zl_llama_finalize(m);
}

extern "C" int zl_llama_set_state(zl_llama_t* m, const int32_t* tokens_host, const int32_t* positions_host,
                                  int B) {
    ZL_CHECK_ARG(m && tokens_host && positions_host && B > 0 && B <= m->cfg.max_batch);
    if (!m->finalized) {
        zl_set_last_error(__FILE__, __LINE__, "model not finalized");
        return ZL_ERR_STATE;
    }
    const int slot = m->ring_next;
    m->ring_next = (slot + 1) % zl_llama::kStageSlots;
    if (m->ring_used[slot]) ZL_CHECK_CUDA(cudaEventSynchronize(m->ring_ev[slot]));   // its previous copies have executed
    int32_t* hs = m->h_ring.get() + (size_t)slot * 2 * m->cfg.max_batch;
    int mx = 0;
    for (int i = 0; i < B; ++i) {
        ZL_CHECK_ARG(positions_host[i] >= 0 && positions_host[i] < m->cfg.max_seq);
        ZL_CHECK_ARG(tokens_host[i] >= 0 && tokens_host[i] < m->cfg.vocab_size);
        hs[i] = tokens_host[i];
        hs[B + i] = positions_host[i];
        if (positions_host[i] + 1 > mx) mx = positions_host[i] + 1;
    }
    m->cur_max_len = mx;
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_tokens.get(), hs, B * 4, cudaMemcpyHostToDevice, m->stream));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_pos.get(), hs + B, B * 4, cudaMemcpyHostToDevice, m->stream));
    ZL_CHECK_CUDA(cudaEventRecord(m->ring_ev[slot], m->stream));
    m->ring_used[slot] = true;
    return ZL_OK;
}

extern "C" int zl_llama_step_device(zl_llama_t* m, int B) {
    ZL_CHECK_ARG(m && B > 0 && B <= m->cfg.max_batch);
    if (m->cur_max_len >= m->cfg.max_seq) {
        zl_set_last_error(__FILE__, __LINE__, "KV buffers full (max_seq reached)");
        return ZL_ERR_STATE;
    }
    RCHECK(run_step(m, B));
    k_advance<<<cdiv(B, 64), 64, 0, m->stream>>>(m->d_tokens.get(), m->d_pos.get(), m->d_next.get(), B, g_w4_trace);
    ZL_CHECK_LAUNCH();
    m->cur_max_len += 1;
    return ZL_OK;
}

extern "C" int zl_llama_decode(zl_llama_t* m, const int32_t* tokens_host, const int32_t* positions_host, int B,
                               int32_t* next_tokens_host, float* logits_host) {
    ZL_CHECK_ARG(next_tokens_host != nullptr);
    RCHECK(zl_llama_set_state(m, tokens_host, positions_host, B));
    RCHECK(run_step(m, B));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->h_stage.get() + 3 * B, m->d_next.get(), B * 4, cudaMemcpyDeviceToHost, m->stream));
    if (logits_host)   // (B, vocab/tp) of this rank's shard
        ZL_CHECK_CUDA(cudaMemcpyAsync(logits_host, m->logits.get(), (size_t)B * m->vshard * 4, cudaMemcpyDeviceToHost,
                                      m->stream));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    for (int i = 0; i < B; ++i) next_tokens_host[i] = m->h_stage.get()[3 * B + i];
    return ZL_OK;
}

extern "C" int zl_llama_get_state(zl_llama_t* m, int32_t* tokens_host, int32_t* positions_host, int B) {
    ZL_CHECK_ARG(m && tokens_host && positions_host && B > 0 && B <= m->cfg.max_batch);
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->h_stage.get(), m->d_tokens.get(), B * 4, cudaMemcpyDeviceToHost, m->stream));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->h_stage.get() + B, m->d_pos.get(), B * 4, cudaMemcpyDeviceToHost, m->stream));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    for (int i = 0; i < B; ++i) {
        tokens_host[i] = m->h_stage.get()[i];
        positions_host[i] = m->h_stage.get()[B + i];
    }
    return ZL_OK;
}

extern "C" int zl_llama_get_logits(zl_llama_t* m, float* logits_host, int B) {
    ZL_CHECK_ARG(m && logits_host && B > 0 && B <= m->cfg.max_batch);
    ZL_CHECK_CUDA(cudaMemcpyAsync(logits_host, m->logits.get(), (size_t)B * m->vshard * 4, cudaMemcpyDeviceToHost, m->stream));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    return ZL_OK;
}

extern "C" int zl_llama_bench_gemms(zl_llama_t* m, int B, int iters, float* ms, int* launches, double* bytes) {
    ZL_CHECK_ARG(m && B > 0 && B <= m->cfg.max_batch && iters > 0 && ms);
    const auto& c = m->cfg;
    const int D = c.dim_model, d = c.dim_head, pdl = c.use_pdl;
    const bool w4 = c.quant_type == 5 || c.quant_type == 6;
    cudaStream_t st = m->stream;
    // the decode step's W4 GEMMs, launched by the same functions (fused RMSNorm, qkv RoPE + KV append, SwiGLU and residual
    // epilogues, PDL policy).  Rewrites the KV rows of the current positions and the residual stream: call it after the
    // measurements that need the decode state.
    Chain ch;
    ch.n = B;
    ch.gemm_only = true;
    ch.h = m->h.get();
    m->cur_tb = m->d_iota.get();
    m->cur_pos = m->d_pos.get();
    cudaEvent_t e0, e1;
    ZL_CHECK_CUDA(cudaEventCreate(&e0));
    ZL_CHECK_CUDA(cudaEventCreate(&e1));
    int n_launch = 0;
    double nbytes = 0;
    for (int it = -1; it < iters; ++it) {   // it == -1: warm-up pass
        if (it == 0) ZL_CHECK_CUDA(cudaEventRecord(e0, st));
        for (int l = 0; l < c.num_layers; ++l) {
            Layer& L = m->layers[l];
            if (w4) {
                RCHECK(qkv_gemm(m, l, ch));
                RCHECK(o_gemm(m, l, ch));
                RCHECK(gate_up_gemm(m, l, ch));
                RCHECK(down_gemm(m, l, ch));
                if (it == 0) {
                    nbytes += (double)zl_w4_packed_bytes(L.q_qkv.N, D, c.group_size) +
                              (double)zl_w4_packed_bytes(D, m->hq * d, c.group_size) +
                              (double)zl_w4_packed_bytes(L.q_gu.N, D, c.group_size) +
                              (double)zl_w4_packed_bytes(D, m->ff, c.group_size);
                    // activations in/out (fp16)
                    nbytes += 2.0 * B * (D + L.q_qkv.N + m->hq * d + 2 * D + D + m->ff + m->ff + 2 * D);
                }
            } else {
                RCHECK(dense_or_w8(m, m->xn.get(), L.d_qkv, m->qkv.get(), B, pdl));
                RCHECK(dense_or_w8(m, m->ao.get(), L.d_o, m->pend.get(), B, pdl));
                RCHECK(dense_or_w8(m, m->xn.get(), L.d_gu, m->gu.get(), B, pdl));
                RCHECK(dense_or_w8(m, m->act.get(), L.d_down, m->pend.get(), B, pdl));
                if (it == 0) {
                    // weight bytes: 2 per element dense, 1 (+ per-row scale) for W8A8 (SURVEY 8d)
                    const double wb = L.d_qkv.w8 ? 1.0 : 2.0;
                    nbytes += wb * ((double)L.d_qkv.N * D + (double)D * m->hq * d + 2.0 * m->ff * D + (double)D * m->ff) +
                              2.0 * B * (D + L.d_qkv.N + m->hq * d + D + D + 2 * m->ff + m->ff + D);
                }
            }
            if (it == 0) n_launch += 4;
        }
    }
    ZL_CHECK_CUDA(cudaEventRecord(e1, st));
    ZL_CHECK_CUDA(cudaEventSynchronize(e1));
    ZL_CHECK_CUDA(cudaEventElapsedTime(ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (launches) *launches = n_launch;
    if (bytes) *bytes = nbytes;
    return ZL_OK;
}

extern "C" int zl_llama_sync(zl_llama_t* m) {
    ZL_CHECK_ARG(m);
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    return ZL_OK;
}

extern "C" int zl_llama_prefill(zl_llama_t* m, int task, const int32_t* tokens_host, int n, int pos0,
                                int32_t* next_token_host, float* logits_host) {
    ZL_CHECK_ARG(m && m->finalized && tokens_host && next_token_host && n > 0 && pos0 >= 0);
    ZL_CHECK_ARG(task >= 0 && task < m->cfg.max_batch);
    const int chunk = m->cfg.prefill_chunk;
    if (chunk <= 0) {
        zl_set_last_error(__FILE__, __LINE__, "zl_llama_prefill needs cfg.prefill_chunk > 0");
        return ZL_ERR_STATE;
    }
    if (pos0 + n > m->cfg.max_seq) {
        zl_set_last_error(__FILE__, __LINE__, "prompt does not fit the KV buffers (max_seq)");
        return ZL_ERR_STATE;
    }
    int32_t* h_tok = m->h_stage.get() + 4 * m->cfg.max_batch + 4;   // pinned staging for one chunk of token ids
    for (int c0 = 0; c0 < n; c0 += chunk) {
        const int cn = (n - c0) < chunk ? (n - c0) : chunk;
        if (c0 > 0) ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));   // staging buffer reuse
        for (int i = 0; i < cn; ++i) {
            ZL_CHECK_ARG(tokens_host[c0 + i] >= 0 && tokens_host[c0 + i] < m->cfg.vocab_size);
            h_tok[i] = tokens_host[c0 + i];
        }
        ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_pf_tokens.get(), h_tok, cn * 4, cudaMemcpyHostToDevice, m->stream));
        Segments pc;
        pc.task = task;
        pc.pos0 = pos0 + c0;
        pc.n = cn;
        pc.last = c0 + cn == n;
        RCHECK(enqueue_step(m, 1, 0, &pc, sampler_on(m, task, 1)));
    }
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->h_stage.get() + 3 * m->cfg.max_batch, m->d_next.get(), 4, cudaMemcpyDeviceToHost, m->stream));
    if (logits_host)
        ZL_CHECK_CUDA(cudaMemcpyAsync(logits_host, m->logits.get(), (size_t)m->vshard * 4, cudaMemcpyDeviceToHost, m->stream));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    *next_token_host = m->h_stage.get()[3 * m->cfg.max_batch];
    if (pos0 + n > m->cur_max_len) m->cur_max_len = pos0 + n;
    return ZL_OK;
}

extern "C" int zl_llama_step_joined(zl_llama_t* m, const int32_t* tokens_host, const int32_t* seg_host, int nseg,
                                    int32_t* next_host, float* logits_host) {
    ZL_CHECK_ARG(m && tokens_host && seg_host && next_host && nseg > 0);
    const auto& c = m->cfg;
    if (c.prefill_chunk <= 0) {
        zl_set_last_error(__FILE__, __LINE__, "zl_llama_step_joined needs cfg.prefill_chunk > 0");
        return ZL_ERR_STATE;
    }
    // zl_varlen_attention reads the activation-dtype cache of one rank
    if (c.kv_int8 || c.tp_size > 1)
        return fail_state(__LINE__, "joined steps are not available with an int8 KV cache or tensor parallelism",
                          ZL_ERR_UNSUPPORTED);
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    ZL_CHECK_ARG(nseg <= c.max_batch);
    // every check before any work is enqueued
    std::vector<char> seen(c.max_batch, 0);
    int rows = 0;
    for (int s = 0; s < nseg; ++s) {
        const int32_t* s4 = seg_host + 4 * s;   // {task, pos0, n, emit}
        ZL_CHECK_ARG(s4[0] >= 0 && s4[0] < c.max_batch && !seen[s4[0]]);
        ZL_CHECK_ARG(s4[2] >= 1 && s4[1] >= 0 && s4[1] <= c.max_seq - s4[2]);
        seen[s4[0]] = 1;
        rows += s4[2];
        ZL_CHECK_ARG(rows <= m->tok_cap);
    }
    for (int i = 0; i < rows; ++i) ZL_CHECK_ARG(tokens_host[i] >= 0 && tokens_host[i] < c.vocab_size);

    // host staging: tokens | positions | token -> task (tok_cap each) | segments | emitting rows | tasks | positions
    const int T = m->tok_cap, MB = c.max_batch;
    int32_t* h_tok = m->h_join.get();
    int32_t* h_pos = h_tok + T;
    int32_t* h_tb = h_pos + T;
    int32_t* h_seg = h_tb + T;
    int32_t* h_erow = h_seg + 4 * MB;
    int32_t* h_etask = h_erow + MB;
    int32_t* h_epos = h_etask + MB;
    Segments sg;
    sg.joined = true;
    sg.n = rows;
    sg.nseg = nseg;
    bool sampler = false;
    for (int s = 0, row0 = 0; s < nseg; ++s) {
        const int task = seg_host[4 * s], pos0 = seg_host[4 * s + 1], n = seg_host[4 * s + 2];
        for (int i = 0; i < n; ++i) {
            h_tok[row0 + i] = tokens_host[row0 + i];
            h_pos[row0 + i] = pos0 + i;
            h_tb[row0 + i] = task;
        }
        h_seg[4 * s] = task;
        h_seg[4 * s + 1] = row0;
        h_seg[4 * s + 2] = pos0;
        h_seg[4 * s + 3] = n;
        if (seg_host[4 * s + 3]) {
            h_erow[sg.n_emit] = row0 + n - 1;
            h_etask[sg.n_emit] = task;
            h_epos[sg.n_emit] = pos0 + n - 1;
            ++sg.n_emit;
            sampler |= m->samp_on[task] != 0;
        }
        if (pos0 + n > sg.max_keys) sg.max_keys = pos0 + n;
        row0 += n;
    }
    cudaStream_t st = m->stream;
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_pf_tokens.get(), h_tok, (size_t)rows * 4, cudaMemcpyHostToDevice, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_pf_pos.get(), h_pos, (size_t)rows * 4, cudaMemcpyHostToDevice, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_tb.get(), h_tb, (size_t)rows * 4, cudaMemcpyHostToDevice, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_join.get(), h_seg, (size_t)7 * MB * 4, cudaMemcpyHostToDevice, st));
    RCHECK(enqueue_step(m, 0, 0, &sg, sampler));
    int32_t* h_next = m->h_stage.get() + 3 * MB;
    if (sg.n_emit) {
        ZL_CHECK_CUDA(cudaMemcpyAsync(h_next, m->d_next.get(), (size_t)sg.n_emit * 4, cudaMemcpyDeviceToHost, st));
        if (logits_host)
            ZL_CHECK_CUDA(cudaMemcpyAsync(logits_host, m->logits.get(), (size_t)sg.n_emit * m->vshard * 4,
                                          cudaMemcpyDeviceToHost, st));
    }
    ZL_CHECK_CUDA(cudaStreamSynchronize(st));   // also frees the pinned staging for the next call
    for (int s = 0, e = 0; s < nseg; ++s) next_host[s] = seg_host[4 * s + 3] ? h_next[e++] : -1;
    if (sg.max_keys > m->cur_max_len) m->cur_max_len = sg.max_keys;
    return ZL_OK;
}

extern "C" int zl_llama_set_sampling(zl_llama_t* m, int task, const zl_sample_params_t* p) {
    if (p) RCHECK(zl_sample_check_params(p, 1));
    ZL_CHECK_ARG(m && task >= 0 && task < m->cfg.max_batch);
    const bool on = p && ((p->temperature > 0.f && p->top_k != 1) || p->repetition_penalty != 1.f ||
                          p->presence_penalty != 0.f);
    ZL_CHECK_SUPPORTED(!on || m->cfg.tp_size == 1);
    if (!m->finalized) {
        zl_set_last_error(__FILE__, __LINE__, "model not finalized");
        return ZL_ERR_STATE;
    }
    const zl_sample_params_t q = p ? *p : zl_sample_params_t{0.f, 1.f, 1.f, 0.f, 0, 0};
    // stream-ordered after every step already enqueued; the pageable source is staged before the call returns
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_sparams.get() + task, &q, sizeof(q), cudaMemcpyHostToDevice, m->stream));
    ZL_CHECK_CUDA(cudaMemsetAsync(m->d_hist.get() + (size_t)task * m->hwords, 0, (size_t)m->hwords * 4, m->stream));
    m->samp_on[task] = on ? 1 : 0;
    return ZL_OK;
}

extern "C" int zl_llama_read_kv(zl_llama_t* m, int layer, int task, int row0, int n, void* k_host, void* v_host,
                                float* sk_host, float* sv_host) {
    ZL_CHECK_ARG(m && m->finalized && layer >= 0 && layer < m->cfg.num_layers && task >= 0 && task < m->cfg.max_batch);
    ZL_CHECK_ARG(row0 >= 0 && n > 0 && row0 + n <= m->cfg.max_seq);
    ZL_CHECK_ARG(m->cfg.kv_int8 || (!sk_host && !sv_host));
    const Layer& L = m->layers[layer];
    const size_t row = (size_t)m->hkv * m->cfg.dim_head;   // values per token
    const size_t vb = m->cfg.kv_int8 ? 1 : 2;               // bytes per value
    const size_t off = ((size_t)task * m->cfg.max_seq + row0) * row * vb;
    const size_t soff = ((size_t)task * m->cfg.max_seq + row0) * m->hkv * 4;
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));   // the steps that wrote the rows
    if (k_host) ZL_CHECK_CUDA(cudaMemcpy(k_host, (char*)L.kbuf.get() + off, n * row * vb, cudaMemcpyDeviceToHost));
    if (v_host) ZL_CHECK_CUDA(cudaMemcpy(v_host, (char*)L.vbuf.get() + off, n * row * vb, cudaMemcpyDeviceToHost));
    if (sk_host) ZL_CHECK_CUDA(cudaMemcpy(sk_host, (char*)L.skbuf.get() + soff, (size_t)n * m->hkv * 4, cudaMemcpyDeviceToHost));
    if (sv_host) ZL_CHECK_CUDA(cudaMemcpy(sv_host, (char*)L.svbuf.get() + soff, (size_t)n * m->hkv * 4, cudaMemcpyDeviceToHost));
    return ZL_OK;
}

extern "C" int zl_llama_config_layout(size_t* size, size_t* kv_int8_offset) {
    ZL_CHECK_ARG(size && kv_int8_offset);
    *size = sizeof(zl_llama_config_t);
    *kv_int8_offset = offsetof(zl_llama_config_t, kv_int8);
    return ZL_OK;
}

extern "C" zl_stream_t zl_llama_stream(zl_llama_t* m) { return m ? (zl_stream_t)m->stream : nullptr; }

extern "C" int zl_llama_stats(zl_llama_t* m, int B, double* weight_bytes, int* kernels_per_step) {
    ZL_CHECK_ARG(m);
    (void)B;
    if (weight_bytes) *weight_bytes = m->weight_bytes;
    if (kernels_per_step) *kernels_per_step = m->kernels_per_step;
    return ZL_OK;
}
