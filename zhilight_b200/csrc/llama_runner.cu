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
#include "kv_pool.cuh"
#include "kv_arena.cuh"
#include "beam.cuh"
#include "sample.cuh"

#include <algorithm>
#include <array>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <numeric>
#include <utility>
#include <string>
#include <vector>

extern unsigned long long* g_w4_trace;   // debug timeline buffer (zl_w4_set_trace)

#define RCHECK(expr)                \
    do {                            \
        int _rc = (expr);           \
        if (_rc != ZL_OK) return _rc; \
    } while (0)

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

// The weight format of a Linear.  lin_format: that of every Linear of a model, by quant_type -- W4A16 GPTQ / AWQ (5, 6;
// 8 is served as 5), dense (0), or W8A8 with int8 rows (2), fp8 rows (7) or fp8 128x128 blocks (10).
enum LinFormat { kW4, kDense, kInt8, kFp8Rows, kFp8Block };
LinFormat lin_format(const zl_llama_config_t& c) {
    switch (c.quant_type) {
        case 5: case 6: return kW4;
        case 2: return kInt8;
        case 7: return kFp8Rows;
        case 10: return kFp8Block;
        default: return kDense;
    }
}

struct Lin {
    LinFormat fmt = kDense;
    int N = 0, K = 0;
    dev_ptr<> bias;
    dev_ptr<> packed;     // W4: ZLW4  (fp16 HMMA kernels) -- only kept when some batch size needs it
    dev_ptr<> packed_i;   // ZLW4I (exact-integer IMMA kernel, small M)
    dev_ptr<int32_t> k_perm;   // act-order: the GEMM reads x[:, k_perm] (K int32); empty: sequential g_idx
    // dense and W8A8: the (N, K) weight, in the activation dtype or as 8-bit codes
    dev_ptr<> w;
    dev_ptr<> w_scale;   // int8: (N) in the activation dtype (linear.cpp:541); fp8: (N) f32 rows;
                         // fp8 block: (N/128, K/128) f32 weight_scale_inv
};

struct Layer {
    dev_ptr<> ln_attn;
    dev_ptr<> ln_ff;
    Lin qkv, o, gu, down;
    dev_ptr<> kbuf;   // the row space (KvArena::rows, Hkv, d): activation dtype, or uint8 codes at kv_int8
    dev_ptr<> vbuf;
    dev_ptr<void*> k_addrs;   // (max_batch): each task's first row, written by the arena (k_kv_relocate)
    dev_ptr<void*> v_addrs;
    dev_ptr<> skbuf;          // kv_int8: (KvArena::rows, Hkv) fp32 scales
    dev_ptr<> svbuf;
    dev_ptr<void*> sk_addrs;  // (max_batch)
    dev_ptr<void*> sv_addrs;
};

// Staging slots for host -> device copies: a pinned copy reads its host slot when it EXECUTES, and a kernel reads its device
// slot when it runs, so a caller that runs ahead of the GPU must not rewrite a slot whose reader is still queued.  kSlots
// slots of `words` int32 each, on the host and (when allocated) on the device, one event each.
struct StageRing {
    static constexpr int kSlots = 8;
    host_ptr<int32_t> h;
    dev_ptr<int32_t> d;
    size_t words = 0;
    cudaEvent_t ev[kSlots] = {};
    bool used[kSlots] = {};
    int next = 0, cur = 0;   // cur: the slot acquire() returned last

    StageRing() = default;
    StageRing(const StageRing&) = delete;
    StageRing& operator=(const StageRing&) = delete;
    ~StageRing() {
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    }
    int alloc(size_t slot_words, bool device);
    // the next slot's host (and device) words, once the reader it was last released to has executed
    int acquire(int32_t** hs, int32_t** ds = nullptr);
    // call after the copy or kernel that reads the acquired slot has been enqueued on st
    int release(cudaStream_t st);
};

// Instantiated graphs by key, destroyed with the cache.  get() returns the graph of `key`, or instantiates and keeps the
// graph build(&graph) makes (the cache owns that graph, also when build fails) and stores its node count in *nodes.
struct GraphCache {
    std::map<long long, cudaGraphExec_t> execs;

    GraphCache() = default;
    GraphCache(const GraphCache&) = delete;
    GraphCache& operator=(const GraphCache&) = delete;
    ~GraphCache() { clear(); }
    void clear() {
        for (auto& g : execs) cudaGraphExecDestroy(g.second);
        execs.clear();
    }
    template <typename Build>
    int get(long long key, Build&& build, cudaGraphExec_t* out, int* nodes = nullptr) {
        auto it = execs.find(key);
        if (it == execs.end()) {
            cudaGraph_t graph = nullptr;
            const int rc = build(&graph);
            std::unique_ptr<CUgraph_st, cudaError_t (*)(cudaGraph_t)> own(graph, cudaGraphDestroy);
            RCHECK(rc);
            cudaGraphExec_t exec = nullptr;
            ZL_CHECK_CUDA(cudaGraphInstantiate(&exec, graph, 0));
            if (nodes) {
                size_t n_nodes = 0;
                cudaGraphGetNodes(graph, nullptr, &n_nodes);
                *nodes = (int)n_nodes;
            }
            it = execs.emplace(key, exec).first;
        }
        *out = it->second;
        return ZL_OK;
    }
};

// Every task's pick state: which parts of the sampler it uses and the sampler's device tables.
//   sampling (zl_llama_set_sampling): parameters and generated-token bitmaps of hwords words
//   logits processors (zl_llama_set_logits_processors): n-gram penalty, bias lists and the generated-token sequence
//     (appended by the sampler where it sets the history bit, cleared with it); the n-gram workspace (k_ngram_levels'
//     tables) is allocated by the first task that turns the n-gram rule on
//   token automata (zl_llama_enable_constraints / zl_llama_set_constraint): au.states mask rows of hwords words, CSR
//     edges (row offsets, tokens, next states), the default next states and the current state (-1: unconstrained)
// `proc` points at the tables as k_sample reads them; a launch sets only its n-gram and frozen fields.
struct TaskPicks {
    enum : uint8_t { kSamples = 1, kProcessors = 2, kNgram = 4, kAutomaton = 8 };
    std::vector<uint8_t> on;   // per task: kSamples (samples or has penalties), kProcessors, kNgram, kAutomaton
    dev_ptr<zl_sample_params_t> params;   // (max_batch)
    dev_ptr<uint32_t> hist;               // (max_batch, hwords)
    int hwords = 0;
    dev_ptr<float> ngram;                 // (max_batch)
    dev_ptr<int32_t> seq, seq_len;        // (max_batch, max_seq), (max_batch)
    dev_ptr<int32_t> bias_tok, bias_cnt;  // (max_batch, ZL_MAX_LOGIT_BIAS), (max_batch)
    dev_ptr<float> bias_val;              // (max_batch, ZL_MAX_LOGIT_BIAS)
    dev_ptr<> ngram_ws;
    dev_ptr<uint32_t> mask;
    dev_ptr<int32_t> row_ptr, edge_tok, edge_next, dflt, state;
    zl::SampleProc proc{};

    int alloc(int B, int vocab, int max_seq, cudaStream_t st);
    int alloc_ngram(int B, int max_seq);
    int alloc_automata(int B, int max_states, int max_edges, cudaStream_t st);
    void set(int t, uint8_t bits, bool v) { on[t] = v ? on[t] | bits : on[t] & ~bits; }
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
    // zl_llama_set_state staging: a set_state -> step_device loop that runs ahead of the GPU must not rewrite a slot whose
    // copies are still queued.  Host slots of 2 * max_batch words.
    StageRing state_ring;
    // prefill keeps its own (token, position) arrays: the decode-state arrays d_tokens / d_pos of tasks 0..B-1 survive a
    // prefill that happens between two zl_llama_step_device calls (continuous batching)
    dev_ptr<int32_t> d_pf_tokens, d_pf_pos;
    zl_comm_t* comm = nullptr;            // TP exchange (set by zl_llama_set_comm when tp_size > 1)
    int vshard = 0;                       // vocabulary rows of lm_head held by this rank
    // tensor parallel: the vocabulary all-gather that gives the sampler and the beam selection whole rows
    // (zl_llama_set_vocab_gather); NULL keeps them refused under tp_size > 1
    zl_vocab_gather_t* vgather = nullptr;
    dev_ptr<> cand;                       // [B] {float value, int index} local argmax candidates
    dev_ptr<> cand_all;                   // [tp][B] gathered candidates
    GraphCache graphs;                    // decode-step graphs, by graph_key (+ the beam bits)
    int cur_max_len = 0;                  // host-side upper bound of buf_lens (positions + 1)
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
    dev_ptr<int8_t> d_mask;   // (chunk, max_seq) causal mask of the chunk
    // joined steps (zl_llama_step_joined): segments {task, row0, pos0, n} for zl_varlen_attention, then per emitting
    // segment its last row | its task | that row's position (max_batch each); h_join stages them with the tokens,
    // positions and token -> task map of the rows (tok_cap each) for the copies into d_pf_tokens / d_pf_pos / d_tb
    dev_ptr<int32_t> d_join;
    host_ptr<int32_t> h_join;
    dev_ptr<> xperm;           // act-order: activations permuted for the GEMM routes that cannot gather (tok_cap x max K)
    // a step whose tasks use none of the sampler runs zl_argmax
    TaskPicks picks;
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
    // where each task's KV rows live (the only owner of task placement), a host mirror of every task's decode position
    // (zl_llama_set_state, step_device, generate) that tells which rows a step writes, and two device tables of 4 entries
    // per layer (K, V, K scales, V scales): the row spaces (kv_bases) and the per-task pointer tables (kv_tabs).  The
    // moves and table entries of a grant are staged in arena_ring slots of 4 * rows / kGrant + max_batch words.
    zl::KvArena arena;
    std::vector<int> pos_host;
    dev_ptr<void*> kv_bases, kv_tabs;
    StageRing arena_ring;
    // prompt prefix cache (zl_llama_kv_pool_create): the device block pool [layer][K|V][block][bt][H_kv][d] (+ fp32 scales
    // [layer][K|V][block][bt][H_kv] at kv_int8), and the block lists of zl_llama_kv_blocks_save / load, staged on the host
    // and the device in slots of 2 * pool_cap words
    dev_ptr<> pool, pool_scales;
    int pool_blocks = 0, pool_bt = 0, pool_cap = 0;   // pool_cap: block pairs one slot holds
    StageRing pool_ring;
    // beam search, allocated by the first zl_llama_beam_step / zl_llama_kv_copy_rows: the selection's inputs and outputs
    // (cum (max_batch) f32 | groups (2 max_batch) | parent, token, score (max_batch x 32) each), its workspace, their
    // pinned host mirror (the beam step is synchronous), and the row-copy ranges staged like the block lists, in slots of
    // 4 * max_batch words
    dev_ptr<> beam_d, beam_ws;
    host_ptr<int32_t> beam_h;
    StageRing rows_ring;
    // generation loop (zl_llama_generate): the per-task stop rules and progress, the loop's control words and the ring of
    // emitted tokens on the device (gen_state lays them out in d_gen), their pinned host mirror, a host mirror of the
    // finish reasons, and one loop graph per (B, sampler, n-gram launch, length bucket), apart from `graphs`
    dev_ptr<int32_t> d_gen;
    host_ptr<int32_t> h_gen;                          // ring rows (max_seq x max_batch) | finish | positions | control
    std::vector<char> gen_fin;
    GraphCache gen_graphs;
};

namespace {

using namespace zl;

template <typename T>
int dmalloc(dev_ptr<T>* p, size_t bytes) {
    void* raw = nullptr;
    ZL_CHECK_CUDA(cudaMalloc(&raw, bytes ? bytes : 16));
    p->reset(static_cast<T*>(raw));
    return ZL_OK;
}

int StageRing::alloc(size_t slot_words, bool device) {
    if (device) RCHECK(dmalloc(&d, sizeof(int32_t) * kSlots * slot_words));
    int32_t* p = nullptr;
    ZL_CHECK_CUDA(cudaMallocHost((void**)&p, sizeof(int32_t) * kSlots * slot_words));
    h.reset(p);
    for (cudaEvent_t& e : ev)
        if (!e) ZL_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    words = slot_words;
    return ZL_OK;
}

int StageRing::acquire(int32_t** hs, int32_t** ds) {
    cur = next;
    next = (cur + 1) % kSlots;
    if (used[cur]) ZL_CHECK_CUDA(cudaEventSynchronize(ev[cur]));   // its previous reader has executed
    *hs = h.get() + (size_t)cur * words;
    if (ds) *ds = d.get() + (size_t)cur * words;
    return ZL_OK;
}

int StageRing::release(cudaStream_t st) {
    ZL_CHECK_CUDA(cudaEventRecord(ev[cur], st));
    used[cur] = true;
    return ZL_OK;
}

// every task greedy, unpenalised, without processors
int TaskPicks::alloc(int B, int vocab, int max_seq, cudaStream_t st) {
    hwords = cdiv(vocab, 32);   // the sampler reads whole rows: the gathered ones under tensor parallelism
    RCHECK(dmalloc(&hist, (size_t)B * hwords * 4));
    ZL_CHECK_CUDA(cudaMemsetAsync(hist.get(), 0, (size_t)B * hwords * 4, st));
    RCHECK(dmalloc(&params, sizeof(zl_sample_params_t) * B));
    {
        const zl_sample_params_t greedy{0.f, 1.f, 1.f, 0.f, 0, 0};
        std::vector<zl_sample_params_t> init(B, greedy);
        ZL_CHECK_CUDA(cudaMemcpyAsync(params.get(), init.data(), sizeof(zl_sample_params_t) * B, cudaMemcpyHostToDevice, st));
        ZL_CHECK_CUDA(cudaStreamSynchronize(st));   // `init` is pageable and goes out of scope
    }
    on.assign(B, 0);
    RCHECK(dmalloc(&ngram, (size_t)B * 4));
    RCHECK(dmalloc(&seq, (size_t)B * max_seq * 4));
    RCHECK(dmalloc(&seq_len, (size_t)B * 4));
    RCHECK(dmalloc(&bias_tok, (size_t)B * ZL_MAX_LOGIT_BIAS * 4));
    RCHECK(dmalloc(&bias_val, (size_t)B * ZL_MAX_LOGIT_BIAS * 4));
    RCHECK(dmalloc(&bias_cnt, (size_t)B * 4));
    ZL_CHECK_CUDA(cudaMemsetAsync(ngram.get(), 0, (size_t)B * 4, st));   // 0.0f: off
    ZL_CHECK_CUDA(cudaMemsetAsync(seq_len.get(), 0, (size_t)B * 4, st));
    ZL_CHECK_CUDA(cudaMemsetAsync(bias_cnt.get(), 0, (size_t)B * 4, st));
    proc = SampleProc{ngram.get(), seq.get(), seq_len.get(), max_seq, bias_tok.get(), bias_val.get(), bias_cnt.get(),
                      ZL_MAX_LOGIT_BIAS, nullptr, ngram_table_size(max_seq)};
    return ZL_OK;
}

// B rows of tables: no launch has more rows than tasks
int TaskPicks::alloc_ngram(int B, int max_seq) {
    RCHECK(dmalloc(&ngram_ws, zl_sample_processed_workspace_bytes(B, max_seq)));
    proc.table = static_cast<int2*>(ngram_ws.get());
    return ZL_OK;
}

int TaskPicks::alloc_automata(int B, int max_states, int max_edges, cudaStream_t st) {
    const size_t S = max_states;
    RCHECK(dmalloc(&mask, B * S * hwords * 4));
    RCHECK(dmalloc(&row_ptr, B * (S + 1) * 4));
    RCHECK(dmalloc(&edge_tok, (size_t)B * max_edges * 4));
    RCHECK(dmalloc(&edge_next, (size_t)B * max_edges * 4));
    RCHECK(dmalloc(&dflt, B * S * 4));
    RCHECK(dmalloc(&state, (size_t)B * 4));
    ZL_CHECK_CUDA(cudaMemsetAsync(state.get(), 0xff, (size_t)B * 4, st));   // -1: unconstrained
    ZL_CHECK_CUDA(cudaStreamSynchronize(st));
    proc.au = SampleAutomata{mask.get(), state.get(), hwords, max_states, max_edges, row_ptr.get(), edge_tok.get(),
                             edge_next.get(), dflt.get()};
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

// drop prefix + suffix for every prefix and suffix
void drop_parts(zl_llama* m, const std::vector<std::string>& prefixes, std::initializer_list<const char*> suffixes) {
    for (const auto& p : prefixes)
        for (const char* s : suffixes) drop(m, p + s);
}

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

// The kernel that serves a W4 Linear at B rows, and what it fuses.
W4Route route_of(const Lin& w, int B) { return w4_route(B, w.N, w.K, 0); }

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
             Lin* out, bool qkv_rope = false, const std::vector<int32_t>* out_rows = nullptr, bool keep_perm = true) {
    const int N = std::accumulate(ns.begin(), ns.end(), 0);
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
    bool need_half = false;
    for (int mm = 1; mm <= (m_max < 17 ? m_max : 17); ++mm)
        if (w4_route(mm, N, K, 0).kernel == W4Kernel::V2) need_half = true;
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
    drop_parts(m, prefixes, {".qweight", ".qzeros", ".scales", ".g_idx", ".bias"});
    out->fmt = kW4;
    out->N = N;
    out->K = K;
    m->weight_bytes += (double)pbytes;
    return ZL_OK;
}

// The part loop of a Linear fused along N from Linears that share its input.  Part i's `prefixes[i].weight` must be
// (ns[i], K) of `elem`-byte elements and, with a PartScale, `prefixes[i] + scale->suffix` must be f32 and pass scale->ok
// (when given); then the weight is copied into `fused` at the part's row offset and scale->copy enqueues what the part's
// scale needs.  A missing or ill-shaped part is reported as "missing/ill-shaped <what> <prefix>".
struct PartScale {
    const char* suffix;
    std::function<bool(size_t i, const Staged& s)> ok;
    std::function<int(size_t i, int off, const Staged& s)> copy;
};

int fuse_parts(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, int K, int elem,
               void* fused, const std::string& what, const PartScale* scale = nullptr) {
    int off = 0;
    for (size_t i = 0; i < prefixes.size(); ++i) {
        const Staged* w = find(m, prefixes[i] + ".weight");
        const Staged* s = scale ? find(m, prefixes[i] + scale->suffix) : nullptr;
        if (!w || w->rows != ns[i] || w->cols != K || w->elem != elem ||
            (scale && (!s || s->elem != 4 || (scale->ok && !scale->ok(i, *s)))))
            return fail_state(__LINE__, "missing/ill-shaped " + what + " " + prefixes[i]);
        ZL_CHECK_CUDA(cudaMemcpyAsync((char*)fused + (size_t)off * K * elem, w->ptr.get(), (size_t)ns[i] * K * elem,
                                      cudaMemcpyDeviceToDevice, m->stream));
        if (scale) RCHECK(scale->copy(i, off, *s));
        off += ns[i];
    }
    return ZL_OK;
}

int build_dense(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, int K, Lin* out) {
    const int N = std::accumulate(ns.begin(), ns.end(), 0);
    RCHECK(dmalloc(&out->w, (size_t)N * K * 2));
    RCHECK(fuse_parts(m, prefixes, ns, K, 2, out->w.get(), "dense weight"));
    RCHECK(build_bias(m, prefixes, ns, &out->bias));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    drop_parts(m, prefixes, {".weight", ".bias"});
    out->fmt = kDense;
    out->N = N;
    out->K = K;
    m->weight_bytes += (double)N * K * 2;
    return ZL_OK;
}

// quant_type 2 (AutoInt8, linear.cpp:521-550): the fp weight is quantised per output row at load with the same kernel
// as the activations; the scale is kept in the activation dtype (functions::typecast, linear.cpp:541).
int dense_to_int8(zl_llama* m, Lin* d) {
    const auto& c = m->cfg;
    dev_ptr<> w8;
    dev_ptr<float> sf;
    RCHECK(dmalloc(&w8, (size_t)d->N * d->K));
    RCHECK(dmalloc(&sf, (size_t)d->N * 4));
    RCHECK(dmalloc(&d->w_scale, (size_t)d->N * 2));
    RCHECK(zl_int8_quant_per_token(d->w.get(), d->K, w8.get(), sf.get(), d->N, d->K, c.dtype, 0, m->stream));
    if (c.dtype == ZL_F16)
        k_f32_to_t<__half><<<cdiv(d->N, 256), 256, 0, m->stream>>>(sf.get(), static_cast<__half*>(d->w_scale.get()), d->N);
    else
        k_f32_to_t<__nv_bfloat16><<<cdiv(d->N, 256), 256, 0, m->stream>>>(
            sf.get(), static_cast<__nv_bfloat16*>(d->w_scale.get()), d->N);
    ZL_CHECK_LAUNCH();
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    d->w = std::move(w8);
    d->fmt = kInt8;
    m->weight_bytes += (double)d->N * d->K + (double)d->N * 2 - (double)d->N * d->K * 2;
    return ZL_OK;
}

// quant_type 7 (Fp8Linear, linear.cpp:1612-1695): e4m3 weights + one f32 weight_scale per Linear.  Projections that
// share an input are fused along N with their scalar scales expanded to one scale per output row.
int build_fp8(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, int K, Lin* out) {
    const int N = std::accumulate(ns.begin(), ns.end(), 0);
    RCHECK(dmalloc(&out->w, (size_t)N * K));
    RCHECK(dmalloc(&out->w_scale, (size_t)N * 4));
    float* w_scale = static_cast<float*>(out->w_scale.get());
    const PartScale expand{".weight_scale", nullptr, [&](size_t i, int off, const Staged& ws) -> int {
                               k_fill_from_scalar<<<cdiv(ns[i], 256), 256, 0, m->stream>>>(
                                   w_scale + off, ns[i], static_cast<const float*>(ws.ptr.get()));
                               ZL_CHECK_LAUNCH();
                               return ZL_OK;
                           }};
    RCHECK(fuse_parts(m, prefixes, ns, K, 1, out->w.get(), "fp8 weight or weight_scale", &expand));
    RCHECK(build_bias(m, prefixes, ns, &out->bias));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    drop_parts(m, prefixes, {".weight", ".weight_scale", ".bias"});
    out->N = N;
    out->K = K;
    out->fmt = kFp8Rows;
    m->weight_bytes += (double)N * K + (double)N * 4;
    return ZL_OK;
}

// quant_type 10 (Fp8Block, linear.cpp:1697-1960): e4m3 weights + weight_scale_inv with one f32 per 128x128 block.
// Projections that share an input are fused along N by concatenating both their weight rows and their scale rows,
// which needs every part's N to be a multiple of 128.  Fp8Block has no bias (set_has_bias throws).
int build_fp8_block(zl_llama* m, const std::vector<std::string>& prefixes, const std::vector<int>& ns, int K,
                    Lin* out) {
    const int N = std::accumulate(ns.begin(), ns.end(), 0);
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
    RCHECK(dmalloc(&out->w, (size_t)N * K));
    RCHECK(dmalloc(&out->w_scale, (size_t)NB * KB * 4));
    char* w_scale = static_cast<char*>(out->w_scale.get());
    const PartScale scale_rows{".weight_scale_inv",
                               [&](size_t i, const Staged& ws) { return ws.rows == (ns[i] + 127) / 128 && ws.cols == KB; },
                               [&](size_t, int off, const Staged& ws) -> int {
                                   ZL_CHECK_CUDA(cudaMemcpyAsync(w_scale + (size_t)(off / 128) * KB * 4, ws.ptr.get(),
                                                                 (size_t)ws.rows * KB * 4, cudaMemcpyDeviceToDevice,
                                                                 m->stream));
                                   return ZL_OK;
                               }};
    RCHECK(fuse_parts(m, prefixes, ns, K, 1, out->w.get(), "fp8 block weight or weight_scale_inv", &scale_rows));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    drop_parts(m, prefixes, {".weight", ".weight_scale_inv"});
    out->N = N;
    out->K = K;
    out->fmt = kFp8Block;
    m->weight_bytes += (double)N * K + (double)NB * KB * 4;
    return ZL_OK;
}

int take_vector(zl_llama* m, const std::string& name, int n, dev_ptr<>* out) {
    auto it = m->staged.find(name);
    if (it == m->staged.end() || (size_t)it->second.rows * it->second.cols != (size_t)n || it->second.elem != 2)
        return fail_state(__LINE__, "missing/ill-shaped tensor " + name);
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
    // the layer's Linears in build order, each fused along N from parts that share its input
    struct Spec {
        std::vector<std::string> prefixes;
        std::vector<int> ns;
        int K;
        Lin* out;
    };
    const Spec lins[] = {
        {{p + "attn.project_q", p + "attn.project_k", p + "attn.project_v"}, {m->hq * d, m->hkv * d, m->hkv * d}, D,
         &L.qkv},
        {{p + "attn.attn_out"}, {D}, m->hq * d, &L.o},
        {{p + "ff.w_in", p + "ff.w_gated"}, {m->ff, m->ff}, D, &L.gu},
        {{p + "ff.w_out"}, {D}, m->ff, &L.down},
    };
    const Spec &qkv = lins[0], &gu = lins[2], &down = lins[3];
    const LinFormat fmt = lin_format(c);
    if (fmt == kW4) {
        // act-order w_out: its permutation orders the gate / up rows, so down runs without one.  A bad w_out g_idx is
        // reported by its own build_w4 below, after the errors of the Linears built before it.
        std::vector<int32_t> down_perm;
        if (g_idx_perm(m, down.prefixes[0], m->ff, &down_perm) != ZL_OK) down_perm.clear();
        for (const Spec& f : lins) {
            const bool swiglu = &f == &gu;
            RCHECK(build_w4(m, f.prefixes, f.ns, f.K, swiglu, f.out, &f == &qkv && c.fuse >= 2,
                            swiglu ? &down_perm : nullptr, &f != &down));
        }
    } else {
        for (const Spec& f : lins) {
            if (fmt == kFp8Rows)
                RCHECK(build_fp8(m, f.prefixes, f.ns, f.K, f.out));
            else if (fmt == kFp8Block)
                RCHECK(build_fp8_block(m, f.prefixes, f.ns, f.K, f.out));
            else
                RCHECK(build_dense(m, f.prefixes, f.ns, f.K, f.out));
        }
        if (fmt == kInt8)
            for (const Spec& f : lins) RCHECK(dense_to_int8(m, f.out));
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

// zl_llama_generate's device state, views of d_gen: per task its stop rule, emitted count, finish reason and the
// last-position bookkeeping; the loop's control words; the ring of emitted tokens
struct GenState {
    int32_t* stop;      // (max_batch, ZL_MAX_STOP_IDS)
    int32_t* n_stop;    // (max_batch) each from here to edge
    int32_t* budget;    // max_new_tokens, 0: none
    int32_t* emitted;   // tokens emitted since the task's last zl_llama_set_stop
    int32_t* fin;       // 0 running, 1 stop id, 2 max_new_tokens, 3 max_seq
    int32_t* ftok;      // a task that filled its KV buffer: the token it fed at max_seq - 1 ...
    int32_t* stok;      // ... and the token it emitted there
    int32_t* edge;      // 1 while such a task re-feeds max_seq - 1 inside a launch
    int32_t* ctl;       // {steps run in this call, steps left in this launch}
    int32_t* ring;      // (max_seq, max_batch): row s = the tokens emitted at step s of the call, -1 where none
    int max_batch, max_seq;
};
constexpr int kGenTaskWords = ZL_MAX_STOP_IDS + 7;   // words per task: stop ids and the seven (max_batch) arrays
constexpr int kGenCtlWords = 4;

GenState gen_state(zl_llama* m) {
    const int MB = m->cfg.max_batch;
    GenState g;
    int32_t* p = m->d_gen.get();
    g.stop = p;
    p += (size_t)MB * ZL_MAX_STOP_IDS;
    for (int32_t** a : {&g.n_stop, &g.budget, &g.emitted, &g.fin, &g.ftok, &g.stok, &g.edge}) {
        *a = p;
        p += MB;
    }
    g.ctl = p;
    g.ring = p + kGenCtlWords;
    g.max_batch = MB;
    g.max_seq = m->cfg.max_seq;
    return g;
}

// every task starts without a stop rule and running
int alloc_generate(zl_llama* m) {
    const auto& c = m->cfg;
    const size_t task_words = (size_t)c.max_batch * kGenTaskWords, ring = (size_t)c.max_seq * c.max_batch;
    RCHECK(dmalloc(&m->d_gen, (task_words + kGenCtlWords + ring) * 4));
    ZL_CHECK_CUDA(cudaMemsetAsync(m->d_gen.get(), 0, (task_words + kGenCtlWords) * 4, m->stream));
    int32_t* h = nullptr;
    ZL_CHECK_CUDA(cudaMallocHost((void**)&h, (ring + 2 * (size_t)c.max_batch + kGenCtlWords) * 4));
    m->h_gen.reset(h);
    m->gen_fin.assign(c.max_batch, 0);
    return ZL_OK;
}

int alloc_runtime(zl_llama* m) {
    const auto& c = m->cfg;
    const int B = c.max_batch, D = c.dim_model, d = c.dim_head;
    // bytes per row: codes (1 byte per value) + one fp32 scale per (token, kv head) at kv_int8, else 2 bytes per value
    const size_t kv_row = (size_t)m->hkv * d * (c.kv_int8 ? 1 : 2);
    const size_t sc_row = (size_t)m->hkv * 4;
    const size_t rows = m->arena.rows;
    // never-written rows must be finite: masked keys still multiply their V rows by an exact 0, and with the dual-stream
    // prefill one half's attention sees the other half's rows before they are appended.  Zero codes with zero scales
    // decode to 0 (the arena zero-fills every row it grants).  The fixed layout's tables point at task t's max_seq rows;
    // an arena's tasks hold no rows yet.
    auto cache = [&](dev_ptr<>* buf, dev_ptr<void*>* tab, size_t row) -> int {
        RCHECK(dmalloc(buf, row * rows));
        ZL_CHECK_CUDA(cudaMemsetAsync(buf->get(), 0, row * rows, m->stream));
        RCHECK(dmalloc(tab, sizeof(void*) * B));
        k_ptr_table<<<cdiv(B, 256), 256, 0, m->stream>>>(tab->get(), (char*)buf->get(),
                                                         m->arena.fixed ? row * c.max_seq : 0, B);
        ZL_CHECK_LAUNCH();
        return ZL_OK;
    };
    std::vector<void*> h_bases, h_tabs;
    for (auto& L : m->layers) {
        RCHECK(cache(&L.kbuf, &L.k_addrs, kv_row));
        RCHECK(cache(&L.vbuf, &L.v_addrs, kv_row));
        if (c.kv_int8) {
            RCHECK(cache(&L.skbuf, &L.sk_addrs, sc_row));
            RCHECK(cache(&L.svbuf, &L.sv_addrs, sc_row));
        }
        for (void* p : {L.kbuf.get(), L.vbuf.get(), L.skbuf.get(), L.svbuf.get()}) h_bases.push_back(p);
        for (void* p : {(void*)L.k_addrs.get(), (void*)L.v_addrs.get(), (void*)L.sk_addrs.get(), (void*)L.sv_addrs.get()})
            h_tabs.push_back(p);
    }
    RCHECK(dmalloc(&m->kv_bases, sizeof(void*) * h_bases.size()));
    RCHECK(dmalloc(&m->kv_tabs, sizeof(void*) * h_tabs.size()));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->kv_bases.get(), h_bases.data(), sizeof(void*) * h_bases.size(),
                                  cudaMemcpyHostToDevice, m->stream));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->kv_tabs.get(), h_tabs.data(), sizeof(void*) * h_tabs.size(), cudaMemcpyHostToDevice,
                                  m->stream));
    if (!m->arena.fixed) RCHECK(m->arena_ring.alloc((size_t)4 * (rows / KvArena::kGrant) + B, true));
    m->pos_host.assign(B, 0);
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
    for (const auto& L : m->layers) act_order |= L.qkv.k_perm || L.o.k_perm || L.gu.k_perm;
    if (act_order) RCHECK(dmalloc(&m->xperm, (size_t)T * (D > m->hq * d ? D : m->hq * d) * 2));
    RCHECK(dmalloc(&m->logits, (size_t)B * c.vocab_size * 4));
    RCHECK(dmalloc(&m->cand, (size_t)((B * 8 + 15) / 16) * 16));
    RCHECK(dmalloc(&m->cand_all, (size_t)((B * 8 + 15) / 16) * 16 * c.tp_size));
    RCHECK(dmalloc(&m->cosb, (size_t)T * d * 4));
    RCHECK(dmalloc(&m->sinb, (size_t)T * d * 4));
    RCHECK(dmalloc(&m->d_tokens, B * 4));
    RCHECK(dmalloc(&m->d_pos, B * 4));
    RCHECK(dmalloc(&m->d_lens, B * 4));
    const LinFormat fmt = lin_format(c);
    if (fmt != kW4 && fmt != kDense) {   // W8A8
        int kmax = D > m->ff ? D : m->ff;
        kmax = kmax > m->hq * d ? kmax : m->hq * d;
        RCHECK(dmalloc(&m->xq, (size_t)T * kmax));
        // fp8 block: one scale per (token, 128 columns), column-major with leading dimension round_up(tokens, 4)
        RCHECK(dmalloc(&m->xs, fmt == kFp8Block ? (size_t)(kmax / 128 + 1) * ((T + 3) / 4 * 4) * 4 : (size_t)T * 4));
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
    RCHECK(m->picks.alloc(B, c.vocab_size, c.max_seq, m->stream));
    RCHECK(alloc_generate(m));
    int32_t* stage = nullptr;
    ZL_CHECK_CUDA(cudaMallocHost((void**)&stage, sizeof(int32_t) * (4 * B + 4 + T)));
    m->h_stage.reset(stage);
    RCHECK(m->state_ring.alloc((size_t)2 * B, false));
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

// The launches of the decode chain, in order.  The stages whose bit (1 << stage) is set in the mask below launch with a
// full dependency instead of a programmatic one (1 qkv GEMM, 2 attention, 4 o GEMM, 8 gate_up GEMM, 16 down GEMM, 32 final
// norm, 64 lm_head, 128 argmax / sampler).
// Single GPU, 66 = lm_head + attention (a PDL-launched lm_head measured much slower): on an
// H100 80GB HBM3 at 400 W, Llama-3.1-8B batch-1 decode measured 425.8 tok/s (425.6-426.2 over 5 runs) against 413.2
// (412.5-415.2) with the o GEMM also fully dependent (70), 420 with attention PDL-launched too (64), and 400-405 with
// lm_head PDL-launched (2, 0)
// (profiles/l2_head_ab.txt): an o GEMM launched early stages its ring fill while attention runs.
// Tensor parallel (exchange inside the GEMMs): 68, a PDL-launched attention kernel measured faster there.
enum Stage { kQkv, kAttn, kO, kGateUp, kDown, kFinalNorm, kLmHead, kPick };

static int stage_pdl(const zl_llama* m, Stage s) {
    const int npm = m->cfg.tp_size > 1 ? 68 : 66;
    return (npm >> s & 1) ? 0 : m->cfg.use_pdl;
}

// the successor of W4 GEMM stage s of layer l in the decode chain -- qkv -> o -> gate_up -> down -> next layer's qkv -- and
// its tensor-parallel mode given this GEMM's (the fused exchange alternates push / reduce-in; the last layer's down keeps
// the stand-alone all-reduce).  The lm_head boundary is left out.
static const Lin* w4_successor(zl_llama* m, int l, Stage s, int tp_mode, int* succ_tp) {
    Layer& L = m->layers[l];
    const bool last = l + 1 >= m->cfg.num_layers;
    *succ_tp = 0;
    switch (s) {
        case kQkv: *succ_tp = tp_mode ? 2 : 0; return &L.o;
        case kO: *succ_tp = tp_mode ? 1 : 0; return &L.gu;
        case kGateUp: *succ_tp = tp_mode && !last ? 2 : 0; return &L.down;
        case kDown: *succ_tp = tp_mode ? 1 : 0; return last ? nullptr : &m->layers[l + 1].qkv;
        default: return nullptr;
    }
}

// row `row` of an fp16 activation matrix of `width` columns
void* rows(const void* base, int row, int width) { return (char*)base + (size_t)row * width * 2; }

// One launch sequence of the layer GEMMs -- a decode step, one half of a dual-stream prefill chunk, or
// zl_llama_bench_gemms -- and the residual stream it updates.
struct Chain {
    // where a W4 o / down GEMM's output goes (dense and W8A8 ones write pend, all-reduced in place at kAllReduce)
    enum Sink {
        kAddResidual,   // o / down add their output to the residual stream in the epilogue
        kPartial,       // o / down write partial sums to pend; the caller reduces them (dual-stream prefill)
        kAllReduce,     // tensor parallel: o / down partial sums -> one-shot all-reduce fused with the residual add
    };
    int row0 = 0, n = 0;       // rows of the activation matrices this sequence covers
    // of the whole launch sequence (index them from row0): its token -> task map (d_iota at decode), positions (d_pos or
    // d_pf_pos) and tokens
    const int32_t* tb = nullptr;
    const int32_t* pos = nullptr;
    const int32_t* tokens = nullptr;
    Sink sink = kAddResidual;
    bool no_pdl = false;       // full dependencies and no L2 head: the next launch is not the chain successor (dual stream)
    bool gemm_only = false;    // launch only what the GEMMs of this fuse level comprise: no stand-alone RMSNorm (fuse 0)
                               // or RoPE / KV append (fuse < 2); dense and W8A8: the GEMM and its activation quant
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
int w4_gemm(zl_llama* m, int l, Stage s, const Chain& ch, const Lin& w, const void* ln_w, zl_w4_fused_args_t a) {
    const auto& c = m->cfg;
    const W4Route route = route_of(w, ch.n);
    const bool half = route.kernel == W4Kernel::V2;   // the fp16 kernel reads the ZLW4 layout
    a.packed = half ? w.packed.get() : w.packed_i.get();
    a.variant = half ? kW4VariantHalf : kW4VariantInt;
    if (!a.packed) return fail_state(__LINE__, "no packed weight variant for this batch size");
    const int pdl = ch.no_pdl ? 0 : c.use_pdl;
    if (ln_w && (c.fuse == 0 || !route.fuses_rmsnorm() || (w.k_perm && !route.gathers_k_perm()))) {
        // the RMSNorm runs as its own kernel (reference order, block.cpp:125,131) into the matching rows of xn: at fuse 0,
        // for the wgmma kernel, which reads x through the TMA engine, and for an act-order GEMM not gathered while staged
        void* xn = rows(m->xn.get(), ch.row0, w.K);
        if (c.fuse > 0 || !ch.gemm_only)
            RCHECK(zl_rmsnorm(a.x, ln_w, xn, ch.n, w.K, c.eps, 1.f, c.dtype, pdl, m->stream));
        a.x = xn;
        ln_w = nullptr;
    }
    if (w.k_perm && route.gathers_k_perm()) {
        a.k_perm = w.k_perm.get();   // gathered while the integer kernel stages x
    } else if (w.k_perm) {
        // the other routes read x in tiles: permute it first (permute_input, gptq/utils.cu:322-398)
        RCHECK(zl_gather_cols_16(a.x, a.ldx, w.k_perm.get(), m->xperm.get(), ch.n, w.K, pdl, m->stream));
        a.x = m->xperm.get();
        a.ldx = w.K;
    }
    W4L2Head l2;
    if (!ch.no_pdl && route.kernel == W4Kernel::V3 && (l2_head_depth() > 0 || l2_whole_max() > 0)) {
        int succ_tp = 0;
        const Lin* nx = w4_successor(m, l, s, a.tp_mode, &succ_tp);
        if (nx && route_of(*nx, ch.n).kernel == W4Kernel::V3)
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
    return zl_kv_int8_quant_append(ks, vs, ch.tb + ch.row0, ch.pos + ch.row0, L.k_addrs.get(), L.v_addrs.get(),
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

// One dense or W8A8 Linear: dense (NormalLinear), or W8A8 = activation quant + fused 8-bit GEMM (Int8Linear::forward /
// Fp8Linear::forward in two launches instead of three)
int dense_or_w8(zl_llama* m, const void* x, const Lin& L, void* y, int B, int pdl) {
    const auto& c = m->cfg;
    cudaStream_t st = m->stream;
    if (L.fmt == kDense) return zl_dense_gemm_skinny(x, L.K, L.w.get(), L.bias.get(), y, B, L.N, L.K, c.dtype, c.dtype, pdl, st);
    if (L.fmt == kInt8) {
        RCHECK(zl_int8_quant_per_token(x, L.K, m->xq.get(), m->xs.get(), B, L.K, c.dtype, pdl, st));
        return zl_w8a8_gemm(m->xq.get(), m->xs.get(), L.w.get(), L.w_scale.get(), c.dtype, L.bias.get(), y, B, L.N, L.K,
                            ZL_W8_INT8, c.dtype, pdl, st);
    }
    if (L.fmt == kFp8Block) {   // Fp8Block::forward: per_token_cast_to_fp8 + the block-scaled GEMM
        const int ld = (B + 3) / 4 * 4;
        RCHECK(zl_fp8_quant_per_token_group(x, L.K, m->xq.get(), m->xs.get(), ld, B, L.K, c.dtype, pdl, st));
        return zl_fp8_block_gemm(m->xq.get(), m->xs.get(), ld, L.w.get(), static_cast<const float*>(L.w_scale.get()), y,
                                 B, L.N, L.K, c.dtype, pdl, st);
    }
    RCHECK(zl_fp8_quant_per_tensor(x, m->xq.get(), m->xs.get(), (size_t)B * L.K, c.dtype, pdl, st));
    return zl_w8a8_gemm(m->xq.get(), m->xs.get(), L.w.get(), L.w_scale.get(), ZL_F32, L.bias.get(), y, B, L.N, L.K,
                        ZL_W8_FP8_ROWS, c.dtype, pdl, st);
}

// Dense and W8A8: the RMSNorm ln of ch's rows of the residual stream into xn, after adding pend_in to them (the previous
// row-parallel Linear's output, or nullptr: block.cpp:139-141 + 131), then the Linear w from xn into y
int dense_norm_gemm(zl_llama* m, const Chain& ch, const void* pend_in, const void* ln, const Lin& w, void* y) {
    const auto& c = m->cfg;
    const int pdl = ch.no_pdl ? 0 : c.use_pdl;
    void* h = rows(ch.h, ch.row0, c.dim_model);
    void* xn = rows(m->xn.get(), ch.row0, c.dim_model);
    if (!ch.gemm_only)
        RCHECK(zl_add_rmsnorm(h, pend_in, ln, h, xn, ch.n, c.dim_model, c.eps, 1.f, 0, c.dtype, pdl, m->stream));
    return dense_or_w8(m, xn, w, y, ch.n, pdl);
}

// qkv: RMSNorm + GEMM; at fuse >= 2 a W4 GEMM's epilogue splits q / k / v, applies RoPE and appends K / V, otherwise
// zl_qkv_rope_append does from the GEMM's output rows a.y.  int8 KV cache: the epilogue appends to the staging rows
// instead (fuse >= 2) or zl_rope_qk_cache writes them (fuse < 2), and kv8_append quantises them into the cache.
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
    const int32_t* tb = ch.tb + ch.row0;
    const int32_t* pos = ch.pos + ch.row0;
    const bool epi = L.qkv.fmt == kW4 && c.fuse >= 2;
    // int8 cache at fuse >= 2 on the exact-integer route (M <= 16): the epilogue quantises K / V into the cache.  The wgmma
    // and fp16 routes, and act-order qkv, append fp16 rows to the staging rows and kv8_append quantises them.
    const bool fused_kv8 = c.kv_int8 && epi && !L.qkv.k_perm && route_of(L.qkv, ch.n).fuses_kv_int8();
    if (epi) {
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
    const int pdl = ch.no_pdl ? 0 : c.use_pdl;
    if (L.qkv.fmt == kW4) {
        ch.reduce_in(&a);
        RCHECK(w4_gemm(m, l, kQkv, ch, L.qkv, L.ln_attn.get(), a));
    } else {
        RCHECK(dense_norm_gemm(m, ch, l == 0 ? nullptr : rows(m->pend.get(), ch.row0, c.dim_model), L.ln_attn.get(), L.qkv,
                               a.y));
    }
    if (ch.gemm_only || fused_kv8) return ZL_OK;
    if (c.kv_int8) return epi ? kv8_append(m, l, ch, pdl) : kv8_rope_append(m, l, ch, a.y, q, pdl);
    if (epi) return ZL_OK;
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

// gate_up: RMSNorm + GEMM + SwiGLU into act: in the W4 GEMM's epilogue, or zl_gate_mul after a dense or W8A8 GEMM
int gate_up_gemm(zl_llama* m, int l, Chain& ch) {
    const auto& c = m->cfg;
    const Layer& L = m->layers[l];
    zl_w4_fused_args_t a = {};
    a.x = rows(ch.h, ch.row0, c.dim_model);
    a.ldx = c.dim_model;
    a.y = rows(m->act.get(), ch.row0, m->ff);
    a.epilogue = ZL_EPI_SWIGLU;
    if (L.gu.fmt != kW4) {
        void* gu = rows(m->gu.get(), ch.row0, 2 * m->ff);
        RCHECK(dense_norm_gemm(m, ch, rows(m->pend.get(), ch.row0, c.dim_model), L.ln_ff.get(), L.gu, gu));
        if (ch.gemm_only) return ZL_OK;
        return zl_gate_mul(gu, 2 * m->ff, (char*)gu + (size_t)m->ff * 2, 2 * m->ff, a.y, m->ff, ch.n, m->ff, 0, c.dtype,
                           m->stream);
    }
    ch.reduce_in(&a);
    return w4_gemm(m, l, kGateUp, ch, L.gu, L.ln_ff.get(), a);
}

// o (input ao) and down (input act): row-parallel under tensor parallelism.  W4: the output goes to ch.sink.  Dense and
// W8A8: it goes to pend, all-reduced in place under tensor parallelism, and the next norm adds it to the residual stream.
int row_parallel_gemm(zl_llama* m, int l, Stage s, Chain& ch) {
    const auto& c = m->cfg;
    const Lin& w = s == kO ? m->layers[l].o : m->layers[l].down;
    const bool w4 = w.fmt == kW4;
    zl_w4_fused_args_t a = {};
    a.x = rows(s == kO ? m->ao.get() : m->act.get(), ch.row0, w.K);
    a.ldx = w.K;
    // the last layer's down keeps the stand-alone all-reduce: the final norm is not a GEMM
    const bool push = w4 && ch.fused && (s == kO || l + 1 < c.num_layers);
    if (push) {
        ch.push(&a);
    } else if (w4 && ch.sink == Chain::kAddResidual) {
        a.residual = a.y = rows(ch.h, ch.row0, c.dim_model);
        a.epilogue = ZL_EPI_RESIDUAL;
    } else {
        a.y = rows(m->pend.get(), ch.row0, c.dim_model);
    }
    const int pdl = ch.no_pdl ? 0 : c.use_pdl;
    RCHECK(w4 ? w4_gemm(m, l, s, ch, w, nullptr, a) : dense_or_w8(m, a.x, w, a.y, ch.n, pdl));
    if (push || ch.gemm_only || ch.sink != Chain::kAllReduce) return ZL_OK;
    return zl_allreduce_one_shot(m->comm, a.y, w4 ? ch.h : nullptr, w4 ? ch.h : a.y, (size_t)ch.n * c.dim_model, c.dtype,
                                 c.tp_int8, pdl, m->stream);
}
int o_gemm(zl_llama* m, int l, Chain& ch) { return row_parallel_gemm(m, l, kO, ch); }
int down_gemm(zl_llama* m, int l, Chain& ch) { return row_parallel_gemm(m, l, kDown, ch); }

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
    if (lin_format(c) != kW4 || c.fuse < 1 || n < 16) return false;
    return force == 1 || (force == 2 && c.tp_size > 1);
}

// ch: the chunk's launch sequence, whose token -> task map, positions and tokens the halves share
int prefill_layers_dual(zl_llama* m, const Segments& pf, const Chain& ch) {
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
        half[h].tb = ch.tb;
        half[h].pos = ch.pos;
        half[h].tokens = ch.tokens;
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

// The pick of a beam step (zl_llama_beam_step): zl_beam_topk's launches over the step's logits, device arguments
struct BeamPick {
    const float* cum = nullptr;
    const int32_t* groups = nullptr;
    int G = 0, K = 0;
    int32_t *parent = nullptr, *token = nullptr;
    float* score = nullptr;
    void* ws = nullptr;
};

// How a launch sequence picks its tokens: zl_argmax (or the tensor-parallel candidate exchange), the sampler -- with the
// n-gram launch when `ngram` -- or a beam step's top-k.  frozen (a loop graph's finish reasons): the sampler records no
// pick of a finished task.
struct Pick {
    bool sampler = false, ngram = false;
    const BeamPick* beam = nullptr;
    const int32_t* frozen = nullptr;

    // task t samples (or has penalties, logits processors or an automaton), and has the n-gram rule on
    void add(const zl_llama* m, int t) {
        sampler |= m->picks.on[t] != 0;
        ngram |= (m->picks.on[t] & TaskPicks::kNgram) != 0;
    }
};

// the sampler and the beam selection can see whole vocabulary rows: a single rank, or the vocabulary all-gather
bool full_rows(const zl_llama* m) { return m->cfg.tp_size == 1 || m->vgather; }

// refuses `what` (with `code`) on a rank that holds only its shard of the vocabulary rows
int need_full_rows(const zl_llama* m, const char* what, int code = ZL_ERR_UNSUPPORTED) {
    if (full_rows(m)) return ZL_OK;
    return fail_state(__LINE__, std::string(what) + " under tensor parallelism needs zl_llama_set_vocab_gather", code);
}

// the pick of tasks first .. first + n - 1
Pick pick_of(const zl_llama* m, int first, int n) {
    Pick pk;
    for (int t = first; t < first + n; ++t) pk.add(m, t);
    return pk;
}

// The final RMSNorm of rows row0 .. row0 + n - 1 of the residual stream h into xn.  W4: the down epilogue already added
// the residual; dense and W8A8: the last down's output (pend) is added here.
int final_norm(zl_llama* m, void* h, int row0, int n, int pdl) {
    const auto& c = m->cfg;
    const int D = c.dim_model;
    void* hr = rows(h, row0, D);
    if (m->layers.back().down.fmt == kW4)
        return zl_rmsnorm(hr, m->ln_f.get(), m->xn.get(), n, D, c.eps, 1.f, c.dtype, pdl, m->stream);
    return zl_add_rmsnorm(hr, rows(m->pend.get(), row0, D), m->ln_f.get(), hr, m->xn.get(), n, D, c.eps, 1.f, 0, c.dtype,
                          pdl, m->stream);
}

int enqueue_step(zl_llama* m, int n_tasks, int len_bucket, const Segments* pf, const Pick& pk) {
    const auto& c = m->cfg;
    const int B = pf ? pf->n : n_tasks;   // rows (tokens) of every activation matrix in this launch sequence
    const int D = c.dim_model, d = c.dim_head, dt = c.dtype, pdl = c.use_pdl;
    cudaStream_t st = m->stream;
    const bool tp = c.tp_size > 1;
    const bool joined = pf && pf->joined;
    if (tp && !m->comm) return fail_state(__LINE__, "tp_size > 1 but zl_llama_set_comm was not called");
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
    Chain ch;
    ch.tb = pf ? m->d_tb.get() : m->d_iota.get();
    ch.pos = pf ? m->d_pf_pos.get() : m->d_pos.get();
    ch.tokens = pf ? m->d_pf_tokens.get() : m->d_tokens.get();
    RCHECK(zl_rope_cos_sin(ch.pos, m->cosb.get(), m->sinb.get(), B, d, c.rope_theta, c.rope_llama3_factor,
                           c.rope_low_freq_factor, c.rope_high_freq_factor, c.rope_orig_ctx, 1, st));
    RCHECK(zl_embedding(ch.tokens, m->emb.get(), m->h.get(), B, D, c.vocab_size, dt, 0, st));
    const bool dual = pf && !joined && prefill_dual_enabled(m, pf->n);
    if (dual) RCHECK(prefill_layers_dual(m, *pf, ch));
    ch.n = B;
    ch.sink = tp ? Chain::kAllReduce : Chain::kAddResidual;
    ch.h = m->h.get();
    ch.ho = m->h2.get();
    // Tensor parallel, decode-sized launches of a W4 model: the exchange rides inside the GEMMs (Chain).  ZL_TP_UNFUSED=1
    // keeps the separate exchange kernels everywhere (A/B).
    ch.fused = tp && lin_format(c) == kW4 && !pf && c.fuse >= 1 && !c.tp_int8 && dt == ZL_F16 && !getenv("ZL_TP_UNFUSED") &&
               (size_t)B * D * 2 <= zl_comm_slot_bytes(m->comm) && 2 * c.num_layers <= 512;
    if (ch.fused) {
        const Layer& L0 = m->layers[0];
        for (const Lin* w : {&L0.qkv, &L0.o, &L0.gu, &L0.down})
            if (!route_of(*w, B).exchanges_tp()) ch.fused = false;
    }
    if (ch.fused) RCHECK(zl_comm_ll_begin_step(m->comm, st));   // the word tags of this step's exchanges
    ch.xodd = ((2 * c.num_layers - 1) & 1) << 9;
    for (int l = 0; l < (dual ? 0 : c.num_layers); ++l) {
        const Layer& L = m->layers[l];
        RCHECK(qkv_gemm(m, l, ch));
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
        RCHECK(o_gemm(m, l, ch));
        RCHECK(gate_up_gemm(m, l, ch));
        RCHECK(down_gemm(m, l, ch));
    }
    const void* head_x = m->xn.get();   // rows that reach lm_head
    if (joined) {
        if (pf->n_emit == 0) return ZL_OK;
        // the final norm is row-wise: norm every row, then gather the emitting segments' last rows into rows
        // 0 .. n_emit - 1 of pend (free after the norm), so that only they reach lm_head
        RCHECK(final_norm(m, m->h.get(), 0, B, pdl));
        k_gather_rows<<<pf->n_emit, 256, 0, st>>>(static_cast<const uint16_t*>(m->xn.get()), j_rows,
                                                 static_cast<uint16_t*>(m->pend.get()), D);
        ZL_CHECK_LAUNCH();
        head_x = m->pend.get();
    } else if (pf) {
        if (!pf->last) return ZL_OK;
        // only the last prompt position feeds the head: move it to row 0 semantics by pointing at its row
        RCHECK(final_norm(m, m->h.get(), pf->n - 1, 1, pdl));
    } else {
        // ch.h: the stream the last exchange left the residual in (h2 after a fused tensor-parallel exchange)
        RCHECK(final_norm(m, ch.h, 0, B, stage_pdl(m, kFinalNorm)));
    }
    const int HB = joined ? pf->n_emit : pf ? 1 : B;   // rows that reach lm_head
    // vocab-parallel lm_head (embedding.cu:353-392): each rank owns vshard rows
    RCHECK(zl_dense_gemm_skinny(head_x, D, m->lm_head, nullptr, m->logits.get(), HB, m->vshard, D, dt, ZL_F32,
                                stage_pdl(m, kLmHead), st));
    // the sampler and the beam selection read whole rows: under tensor parallelism every rank gathers the shards and
    // picks the same tokens from the same rows (both are deterministic), so no pick is broadcast
    const float* rows_v = m->logits.get();
    if (tp && (pk.beam || pk.sampler)) {
        RCHECK(need_full_rows(m, "a sampled or beam pick", ZL_ERR_STATE));
        RCHECK(zl_vocab_allgather(m->vgather, m->logits.get(), HB, m->vshard, pdl, st));
        rows_v = zl_vocab_gather_buffer(m->vgather);
    }
    if (const BeamPick* beam = pk.beam) {
        // decode rows only, no sampling (zl_llama_beam_step checks)
        RCHECK(beam_topk_launch(rows_v, HB, c.vocab_size, beam->cum, beam->groups, beam->G, beam->K, beam->parent,
                                beam->token, beam->score, beam->ws, stage_pdl(m, kPick), st));
    } else if (pk.sampler) {
        // one row per task at decode (row b = task b, counter = its input position); prefill: the task's last prompt
        // position; joined: each emitting segment's task and last position
        const int32_t* row_task = joined ? j_task : pf ? m->d_iota.get() + pf->task : m->d_iota.get();
        const int32_t* counter = joined ? j_pos : pf ? m->d_pf_pos.get() + (pf->n - 1) : m->d_pos.get();
        // k_ngram_levels runs only when a task of the step has the n-gram rule on (`pk.ngram`, a bit of the graph key)
        // with automata enabled every sampler launch reads the tasks' states (-1: unconstrained), so no key bit is needed
        SampleProc pr = m->picks.proc;
        if (!pk.ngram) {
            pr.ngram = nullptr;
            pr.table = nullptr;
        }
        pr.frozen = pk.frozen;
        RCHECK(sample_launch(rows_v, HB, c.vocab_size, m->picks.params.get(), row_task, counter, m->picks.hist.get(),
                             m->picks.hwords, pr, m->d_next.get(), stage_pdl(m, kPick), st));
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

// The key bits the step and loop graphs share: B (bits 33 ..), the sampler (bit 32), the n-gram launch (bit 31) and the
// length bucket (below 2^31).  Parameter changes need no re-capture (they live on the device), only switching the sampler
// or the n-gram launch on or off does.
long long graph_key(int B, const Pick& pk, int bucket) {
    return ((long long)B << 33) | ((long long)pk.sampler << 32) | ((long long)pk.ngram << 31) | (unsigned)bucket;
}

int run_step(zl_llama* m, int B, const BeamPick* beam = nullptr) {
    const int bucket = len_bucket_of(m, m->cur_max_len);
    Pick pk = pick_of(m, 0, B);
    pk.beam = beam;
    if (!m->cfg.use_graph) return enqueue_step(m, B, bucket, nullptr, pk);
    // a beam step (bit 62) bakes its group count (bits 44-54) and K (bits 55-60) into its launches; B < 2048 at a beam step
    long long key = graph_key(B, pk, bucket);
    if (beam) key |= (1LL << 62) | ((long long)beam->K << 55) | ((long long)beam->G << 44);
    auto capture = [&](cudaGraph_t* graph) -> int {
        ZL_CHECK_CUDA(cudaStreamBeginCapture(m->stream, cudaStreamCaptureModeThreadLocal));
        const int rc = enqueue_step(m, B, bucket, nullptr, pk);
        const cudaError_t ce = cudaStreamEndCapture(m->stream, graph);
        RCHECK(rc);
        ZL_CHECK_CUDA(ce);
        return ZL_OK;
    };
    cudaGraphExec_t exec = nullptr;
    RCHECK(m->graphs.get(key, capture, &exec, &m->kernels_per_step));
    ZL_CHECK_CUDA(cudaGraphLaunch(exec, m->stream));
    return ZL_OK;
}

// The pick readback: the n picks in d_next and, when logits_host is given, their n logits rows, once everything enqueued
// has executed.  *picks: the picks in the pinned staging words.
int read_picks(zl_llama* m, int n, float* logits_host, const int32_t** picks) {
    int32_t* h = m->h_stage.get() + 3 * m->cfg.max_batch;
    cudaStream_t st = m->stream;
    if (n > 0) {
        ZL_CHECK_CUDA(cudaMemcpyAsync(h, m->d_next.get(), (size_t)n * 4, cudaMemcpyDeviceToHost, st));
        if (logits_host)   // (n, vocab/tp) of this rank's shard
            ZL_CHECK_CUDA(cudaMemcpyAsync(logits_host, m->logits.get(), (size_t)n * m->vshard * 4, cudaMemcpyDeviceToHost,
                                          st));
    }
    ZL_CHECK_CUDA(cudaStreamSynchronize(st));
    *picks = h;
    return ZL_OK;
}

// Before work that writes (or reads) rows [0, rows) of each {task, rows} of `needs`: grants the rows the tasks lack from
// the arena and enqueues the relocation -- k_kv_relocate launches in order, the last one rewriting the per-task tables.
// ZL_ERR_KV_FULL when they cannot all be granted; then nothing is enqueued and no task moves.  The host arena takes the
// new placement only once every launch is enqueued.  A CUDA error between the first launch and the last leaves rows
// partly moved and the tables not yet rewritten: the model must then be destroyed, as after any CUDA error of a step.
int kv_reserve(zl_llama* m, const std::vector<std::pair<int, int>>& needs) {
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    std::vector<std::vector<KvMove>> launches;
    KvArena next;
    const int rc = m->arena.plan(needs, &next, &launches);
    if (rc == ZL_ERR_KV_FULL)
        return fail_state(__LINE__, "the KV arena cannot grant the rows this call writes (release a task, or a smaller call)",
                          ZL_ERR_KV_FULL);
    RCHECK(rc);
    if (launches.empty()) return ZL_OK;
    const auto& c = m->cfg;
    const int MB = c.max_batch;
    // a launch holds at most rows / kGrant moves (their destinations are disjoint multiples of kGrant rows)
    for (const std::vector<KvMove>& mv : launches)
        if (4 * mv.size() + MB > m->arena_ring.words) return fail_state(__LINE__, "KV arena move list overflows its slot");
    for (size_t i = 0; i < launches.size(); ++i) {
        const std::vector<KvMove>& mv = launches[i];
        const bool last = i + 1 == launches.size();
        int32_t *hs = nullptr, *ds = nullptr;
        RCHECK(m->arena_ring.acquire(&hs, &ds));
        int max_rows = 0;
        for (size_t j = 0; j < mv.size(); ++j) {
            std::memcpy(hs + 4 * j, &mv[j], sizeof(KvMove));
            max_rows = std::max(max_rows, mv[j].copy + mv[j].zero);
        }
        if (last) std::memcpy(hs + 4 * mv.size(), next.first.data(), sizeof(int32_t) * MB);
        ZL_CHECK_CUDA(cudaMemcpyAsync(ds, hs, sizeof(int32_t) * (4 * mv.size() + (last ? MB : 0)), cudaMemcpyHostToDevice,
                                      m->stream));
        KvRelocateArgs a{};
        a.bases = m->kv_bases.get();
        a.moves = ds;
        a.n = (int)mv.size();
        a.layers = c.num_layers;
        a.max_rows = max_rows;
        a.row_bytes = m->hkv * c.dim_head * (c.kv_int8 ? 1 : 2);
        a.srow_bytes = c.kv_int8 ? m->hkv * 4 : 0;
        if (last) {
            a.tabs = reinterpret_cast<void** const*>(m->kv_tabs.get());
            a.firsts = ds + 4 * mv.size();
            a.n_tasks = MB;
        }
        RCHECK(kv_relocate(a, m->stream));
        RCHECK(m->arena_ring.release(m->stream));
    }
    m->arena = std::move(next);
    return ZL_OK;
}

// the rows a decode step of tasks 0 .. B-1 at `positions` writes: row p of each task
int kv_reserve_step(zl_llama* m, const int* positions, int B) {
    std::vector<std::pair<int, int>> needs(B);
    for (int i = 0; i < B; ++i) needs[i] = {i, std::min(positions[i] + 1, m->cfg.max_seq)};
    return kv_reserve(m, needs);
}

// every check of zl_llama_set_state's arguments
int check_state(const zl_llama* m, const int32_t* tokens_host, const int32_t* positions_host, int B) {
    ZL_CHECK_ARG(m && tokens_host && positions_host && B > 0 && B <= m->cfg.max_batch);
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    for (int i = 0; i < B; ++i) {
        ZL_CHECK_ARG(positions_host[i] >= 0 && positions_host[i] < m->cfg.max_seq);
        ZL_CHECK_ARG(tokens_host[i] >= 0 && tokens_host[i] < m->cfg.vocab_size);
    }
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
    ZL_CHECK_SUPPORTED(lin_format(*cfg) != kW4 || cfg->dtype == ZL_F16);
    ZL_CHECK_SUPPORTED(!(cfg->quant_type == 2 || cfg->quant_type == 7) || cfg->tp_size == 1);   // "A must be half" q_gemm_k_major.cu:989
    ZL_CHECK_SUPPORTED(cfg->dtype == ZL_F16 || cfg->dtype == ZL_BF16);
    ZL_CHECK_SUPPORTED(cfg->tp_size >= 1 && cfg->tp_rank >= 0 && cfg->tp_rank < cfg->tp_size);
    ZL_CHECK_SUPPORTED(cfg->num_heads % cfg->tp_size == 0 && cfg->num_kv_heads % cfg->tp_size == 0 &&
                       cfg->dim_ff % cfg->tp_size == 0 && cfg->vocab_size % cfg->tp_size == 0);
    ZL_CHECK_SUPPORTED(lin_format(*cfg) != kW4 || cfg->group_size == zl::kW4GroupK);
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
    zl::KvArena arena;
    if (arena.init(cfg->kv_rows, cfg->max_batch, cfg->max_seq) != ZL_OK)
        return fail_state(__LINE__, "kv_rows must be 0 (fixed layout) or 1 .. max_batch * max_seq", ZL_ERR_INVALID_ARG);
    RCHECK(zl_prepare());
    zl_llama* m = new zl_llama();
    m->cfg = *cfg;
    m->arena = std::move(arena);
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

extern "C" int zl_llama_set_vocab_gather(zl_llama_t* m, zl_vocab_gather_t* g) {
    ZL_CHECK_ARG(m && g);
    int rank = 0, ws = 0, max_rows = 0, vocab = 0;
    RCHECK(zl_vocab_gather_info(g, &rank, &ws, &max_rows, &vocab));
    // at most max_batch rows reach lm_head: a decode or beam step's tasks, a prefill's last position, a joined step's
    // emitting segments
    ZL_CHECK_ARG(ws == m->cfg.tp_size && rank == m->cfg.tp_rank && max_rows >= m->cfg.max_batch &&
                 vocab == m->cfg.vocab_size);
    m->vgather = g;
    return ZL_OK;
}

extern "C" void zl_llama_destroy(zl_llama_t* m) {
    if (!m) return;
    cudaStreamSynchronize(m->stream);
    if (m->reduce_stream) cudaStreamSynchronize(m->reduce_stream);
    for (int h = 0; h < 2; ++h)
        for (cudaEvent_t e : {m->ev_o[h], m->ev_r1[h], m->ev_dn[h], m->ev_r2[h]})
            if (e) cudaEventDestroy(e);
    if (m->reduce_stream) cudaStreamDestroy(m->reduce_stream);
    cudaStreamDestroy(m->stream);
    delete m;   // the members free their device and pinned buffers, graphs and staging events
}

extern "C" int zl_llama_load_tensor(zl_llama_t* m, const char* name, const void* data_host, int rows, int cols,
                                    int elem_bytes) {
    ZL_CHECK_ARG(m && name && data_host && rows > 0 && cols > 0 && elem_bytes > 0);
    if (m->finalized) return fail_state(__LINE__, "model already finalized");
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
    if (m->finalized) return fail_state(__LINE__, "model already finalized");
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
    RCHECK(check_state(m, tokens_host, positions_host, B));
    int32_t* hs = nullptr;
    RCHECK(m->state_ring.acquire(&hs));
    int mx = 0;
    for (int i = 0; i < B; ++i) {
        hs[i] = tokens_host[i];
        hs[B + i] = positions_host[i];
        m->pos_host[i] = positions_host[i];
        if (positions_host[i] + 1 > mx) mx = positions_host[i] + 1;
    }
    m->cur_max_len = mx;
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_tokens.get(), hs, B * 4, cudaMemcpyHostToDevice, m->stream));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_pos.get(), hs + B, B * 4, cudaMemcpyHostToDevice, m->stream));
    return m->state_ring.release(m->stream);
}

extern "C" int zl_llama_step_device(zl_llama_t* m, int B) {
    ZL_CHECK_ARG(m && B > 0 && B <= m->cfg.max_batch);
    if (m->cur_max_len >= m->cfg.max_seq) return fail_state(__LINE__, "KV buffers full (max_seq reached)");
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    RCHECK(kv_reserve_step(m, m->pos_host.data(), B));
    RCHECK(run_step(m, B));
    k_advance<<<cdiv(B, 64), 64, 0, m->stream>>>(m->d_tokens.get(), m->d_pos.get(), m->d_next.get(), B, g_w4_trace);
    ZL_CHECK_LAUNCH();
    for (int i = 0; i < B; ++i) m->pos_host[i] += 1;
    m->cur_max_len += 1;
    return ZL_OK;
}

extern "C" int zl_llama_decode(zl_llama_t* m, const int32_t* tokens_host, const int32_t* positions_host, int B,
                               int32_t* next_tokens_host, float* logits_host) {
    ZL_CHECK_ARG(next_tokens_host != nullptr);
    RCHECK(check_state(m, tokens_host, positions_host, B));
    RCHECK(kv_reserve_step(m, positions_host, B));
    RCHECK(zl_llama_set_state(m, tokens_host, positions_host, B));
    RCHECK(run_step(m, B));
    const int32_t* picks = nullptr;
    RCHECK(read_picks(m, B, logits_host, &picks));
    for (int i = 0; i < B; ++i) next_tokens_host[i] = picks[i];
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
    RCHECK(kv_reserve_step(m, m->pos_host.data(), B));
    const auto& c = m->cfg;
    const int D = c.dim_model, d = c.dim_head;
    cudaStream_t st = m->stream;
    // the decode step's layer GEMMs, launched by the same stage functions (W4: fused RMSNorm, qkv RoPE + KV append, SwiGLU
    // and residual epilogues, PDL policy; W8A8: with the activation quantisation).  Rewrites the KV rows of the current
    // positions and the residual stream: call it after the measurements that need the decode state.
    Chain ch;
    ch.n = B;
    ch.gemm_only = true;
    ch.h = m->h.get();
    ch.tb = m->d_iota.get();
    ch.pos = m->d_pos.get();
    cudaEvent_t e0, e1;
    ZL_CHECK_CUDA(cudaEventCreate(&e0));
    ZL_CHECK_CUDA(cudaEventCreate(&e1));
    int n_launch = 0;
    double nbytes = 0;
    for (int it = -1; it < iters; ++it) {   // it == -1: warm-up pass
        if (it == 0) ZL_CHECK_CUDA(cudaEventRecord(e0, st));
        for (int l = 0; l < c.num_layers; ++l) {
            RCHECK(qkv_gemm(m, l, ch));
            RCHECK(o_gemm(m, l, ch));
            RCHECK(gate_up_gemm(m, l, ch));
            RCHECK(down_gemm(m, l, ch));
            if (it != 0) continue;
            const Layer& L = m->layers[l];
            n_launch += 4;
            if (L.qkv.fmt == kW4) {
                nbytes += (double)zl_w4_packed_bytes(L.qkv.N, D, c.group_size) +
                          (double)zl_w4_packed_bytes(D, m->hq * d, c.group_size) +
                          (double)zl_w4_packed_bytes(L.gu.N, D, c.group_size) +
                          (double)zl_w4_packed_bytes(D, m->ff, c.group_size);
                // activations in/out (fp16)
                nbytes += 2.0 * B * (D + L.qkv.N + m->hq * d + 2 * D + D + m->ff + m->ff + 2 * D);
            } else {
                // weight bytes: 2 per element dense, 1 (+ per-row scale) for W8A8 (SURVEY 8d)
                const double wb = L.qkv.fmt == kDense ? 2.0 : 1.0;
                nbytes += wb * ((double)L.qkv.N * D + (double)D * m->hq * d + 2.0 * m->ff * D + (double)D * m->ff) +
                          2.0 * B * (D + L.qkv.N + m->hq * d + D + D + 2 * m->ff + m->ff + D);
            }
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
    if (chunk <= 0) return fail_state(__LINE__, "zl_llama_prefill needs cfg.prefill_chunk > 0");
    if (pos0 + n > m->cfg.max_seq) return fail_state(__LINE__, "prompt does not fit the KV buffers (max_seq)");
    for (int i = 0; i < n; ++i) ZL_CHECK_ARG(tokens_host[i] >= 0 && tokens_host[i] < m->cfg.vocab_size);
    RCHECK(kv_reserve(m, {{task, pos0 + n}}));
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
        RCHECK(enqueue_step(m, 1, 0, &pc, pick_of(m, task, 1)));
    }
    const int32_t* picks = nullptr;
    RCHECK(read_picks(m, 1, logits_host, &picks));
    *next_token_host = picks[0];
    if (pos0 + n > m->cur_max_len) m->cur_max_len = pos0 + n;
    return ZL_OK;
}

extern "C" int zl_llama_step_joined(zl_llama_t* m, const int32_t* tokens_host, const int32_t* seg_host, int nseg,
                                    int32_t* next_host, float* logits_host) {
    ZL_CHECK_ARG(m && tokens_host && seg_host && next_host && nseg > 0);
    const auto& c = m->cfg;
    if (c.prefill_chunk <= 0) return fail_state(__LINE__, "zl_llama_step_joined needs cfg.prefill_chunk > 0");
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
    std::vector<std::pair<int, int>> needs(nseg);
    for (int s = 0; s < nseg; ++s) needs[s] = {seg_host[4 * s], seg_host[4 * s + 1] + seg_host[4 * s + 2]};
    RCHECK(kv_reserve(m, needs));

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
    Pick pk;   // of the emitting tasks
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
            pk.add(m, task);
        }
        if (pos0 + n > sg.max_keys) sg.max_keys = pos0 + n;
        row0 += n;
    }
    cudaStream_t st = m->stream;
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_pf_tokens.get(), h_tok, (size_t)rows * 4, cudaMemcpyHostToDevice, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_pf_pos.get(), h_pos, (size_t)rows * 4, cudaMemcpyHostToDevice, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_tb.get(), h_tb, (size_t)rows * 4, cudaMemcpyHostToDevice, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->d_join.get(), h_seg, (size_t)7 * MB * 4, cudaMemcpyHostToDevice, st));
    RCHECK(enqueue_step(m, 0, 0, &sg, pk));
    const int32_t* picks = nullptr;
    RCHECK(read_picks(m, sg.n_emit, logits_host, &picks));   // also frees the pinned staging for the next call
    for (int s = 0, e = 0; s < nseg; ++s) next_host[s] = seg_host[4 * s + 3] ? picks[e++] : -1;
    if (sg.max_keys > m->cur_max_len) m->cur_max_len = sg.max_keys;
    return ZL_OK;
}

extern "C" int zl_llama_set_sampling(zl_llama_t* m, int task, const zl_sample_params_t* p) {
    if (p) RCHECK(zl_sample_check_params(p, 1));
    ZL_CHECK_ARG(m && task >= 0 && task < m->cfg.max_batch);
    const bool on = p && ((p->temperature > 0.f && p->top_k != 1) || p->repetition_penalty != 1.f ||
                          p->presence_penalty != 0.f);
    if (on) RCHECK(need_full_rows(m, "zl_llama_set_sampling"));
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    TaskPicks& picks = m->picks;
    const zl_sample_params_t q = p ? *p : zl_sample_params_t{0.f, 1.f, 1.f, 0.f, 0, 0};
    // stream-ordered after every step already enqueued; the pageable source is staged before the call returns
    ZL_CHECK_CUDA(cudaMemcpyAsync(picks.params.get() + task, &q, sizeof(q), cudaMemcpyHostToDevice, m->stream));
    ZL_CHECK_CUDA(cudaMemsetAsync(picks.hist.get() + (size_t)task * picks.hwords, 0, (size_t)picks.hwords * 4, m->stream));
    ZL_CHECK_CUDA(cudaMemsetAsync(picks.seq_len.get() + task, 0, 4, m->stream));
    picks.set(task, TaskPicks::kSamples, on);
    return ZL_OK;
}

extern "C" int zl_llama_set_logits_processors(zl_llama_t* m, int task, float ngram_penalty, const int32_t* bias_tokens_host,
                                              const float* bias_values_host, int n_bias) {
    ZL_CHECK_ARG(m && task >= 0 && task < m->cfg.max_batch);
    ZL_CHECK_ARG(ngram_penalty > 0.f && ngram_penalty < INFINITY);
    ZL_CHECK_ARG(n_bias >= 0 && n_bias <= ZL_MAX_LOGIT_BIAS);
    ZL_CHECK_ARG(n_bias == 0 || (bias_tokens_host && bias_values_host));
    std::vector<int32_t> sorted(bias_tokens_host, bias_tokens_host + n_bias);
    for (int i = 0; i < n_bias; ++i) {
        ZL_CHECK_ARG(bias_tokens_host[i] >= 0 && bias_tokens_host[i] < m->cfg.vocab_size);
        ZL_CHECK_ARG(bias_values_host[i] < INFINITY);   // finite or -inf: NaN and +inf fail
    }
    std::sort(sorted.begin(), sorted.end());
    ZL_CHECK_ARG(std::adjacent_find(sorted.begin(), sorted.end()) == sorted.end());
    const bool ngram = ngram_penalty > 1.f, on = ngram || n_bias > 0;
    if (on) RCHECK(need_full_rows(m, "zl_llama_set_logits_processors"));
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    TaskPicks& picks = m->picks;
    if (ngram && !picks.ngram_ws) RCHECK(picks.alloc_ngram(m->cfg.max_batch, m->cfg.max_seq));
    // stream-ordered after every step already enqueued; pageable sources are staged before the copies return
    cudaStream_t st = m->stream;
    ZL_CHECK_CUDA(cudaMemcpyAsync(picks.ngram.get() + task, &ngram_penalty, 4, cudaMemcpyHostToDevice, st));
    if (n_bias > 0) {
        ZL_CHECK_CUDA(cudaMemcpyAsync(picks.bias_tok.get() + (size_t)task * ZL_MAX_LOGIT_BIAS, bias_tokens_host,
                                      (size_t)n_bias * 4, cudaMemcpyHostToDevice, st));
        ZL_CHECK_CUDA(cudaMemcpyAsync(picks.bias_val.get() + (size_t)task * ZL_MAX_LOGIT_BIAS, bias_values_host,
                                      (size_t)n_bias * 4, cudaMemcpyHostToDevice, st));
    }
    ZL_CHECK_CUDA(cudaMemcpyAsync(picks.bias_cnt.get() + task, &n_bias, 4, cudaMemcpyHostToDevice, st));
    picks.set(task, TaskPicks::kProcessors, on);
    picks.set(task, TaskPicks::kNgram, ngram);
    return ZL_OK;
}

extern "C" int zl_llama_enable_constraints(zl_llama_t* m, int max_states, int max_edges) {
    ZL_CHECK_ARG(m && max_states >= 1 && max_edges >= 0);
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    if (m->picks.mask) return fail_state(__LINE__, "zl_llama_enable_constraints was already called");
    RCHECK(m->picks.alloc_automata(m->cfg.max_batch, max_states, max_edges, m->stream));
    // the sampler launches captured so far carry no automata
    m->graphs.clear();
    m->gen_graphs.clear();
    return ZL_OK;
}

extern "C" int zl_llama_set_constraint(zl_llama_t* m, int task, int n_states, const uint32_t* masks_host,
                                       const int32_t* row_ptr_host, int n_edges, const int32_t* edge_tok_host,
                                       const int32_t* edge_next_host, const int32_t* default_next_host, int start) {
    ZL_CHECK_ARG(m && task >= 0 && task < m->cfg.max_batch && n_states >= 0);
    TaskPicks& picks = m->picks;
    const int W = picks.hwords, S = n_states;
    if (S > 0) RCHECK(need_full_rows(m, "zl_llama_set_constraint"));
    if (!picks.mask) return fail_state(__LINE__, "zl_llama_set_constraint needs zl_llama_enable_constraints");
    if (S > 0) {
        ZL_CHECK_ARG(S <= picks.proc.au.states && n_edges >= 0 && n_edges <= picks.proc.au.max_edges);
        RCHECK(zl_token_automaton_check(m->cfg.vocab_size, S, masks_host, row_ptr_host, n_edges, edge_tok_host,
                                        edge_next_host, default_next_host, start));
    }
    // stream-ordered after every step already enqueued; pageable sources are staged before the copies return
    cudaStream_t st = m->stream;
    const size_t MS = picks.proc.au.states, ME = picks.proc.au.max_edges;
    const int32_t state = S > 0 ? start : -1;
    if (S > 0) {
        ZL_CHECK_CUDA(cudaMemcpyAsync(picks.mask.get() + task * MS * W, masks_host, (size_t)S * W * 4,
                                      cudaMemcpyHostToDevice, st));
        ZL_CHECK_CUDA(cudaMemcpyAsync(picks.row_ptr.get() + task * (MS + 1), row_ptr_host, (size_t)(S + 1) * 4,
                                      cudaMemcpyHostToDevice, st));
        ZL_CHECK_CUDA(cudaMemcpyAsync(picks.dflt.get() + task * MS, default_next_host, (size_t)S * 4,
                                      cudaMemcpyHostToDevice, st));
        if (n_edges > 0) {
            ZL_CHECK_CUDA(cudaMemcpyAsync(picks.edge_tok.get() + task * ME, edge_tok_host, (size_t)n_edges * 4,
                                          cudaMemcpyHostToDevice, st));
            ZL_CHECK_CUDA(cudaMemcpyAsync(picks.edge_next.get() + task * ME, edge_next_host, (size_t)n_edges * 4,
                                          cudaMemcpyHostToDevice, st));
        }
    }
    ZL_CHECK_CUDA(cudaMemcpyAsync(picks.state.get() + task, &state, 4, cudaMemcpyHostToDevice, st));
    picks.set(task, TaskPicks::kAutomaton, S > 0);
    return ZL_OK;
}

extern "C" int zl_llama_get_constraint_state(zl_llama_t* m, int32_t* states_host, int B) {
    ZL_CHECK_ARG(m && states_host && B > 0 && B <= m->cfg.max_batch);
    if (!m->picks.mask) return fail_state(__LINE__, "zl_llama_get_constraint_state needs zl_llama_enable_constraints");
    ZL_CHECK_CUDA(cudaMemcpyAsync(m->h_stage.get(), m->picks.state.get(), (size_t)B * 4, cudaMemcpyDeviceToHost, m->stream));
    ZL_CHECK_CUDA(cudaStreamSynchronize(m->stream));
    for (int i = 0; i < B; ++i) states_host[i] = m->h_stage.get()[i];
    return ZL_OK;
}

extern "C" int zl_llama_read_kv(zl_llama_t* m, int layer, int task, int row0, int n, void* k_host, void* v_host,
                                float* sk_host, float* sv_host) {
    ZL_CHECK_ARG(m && m->finalized && layer >= 0 && layer < m->cfg.num_layers && task >= 0 && task < m->cfg.max_batch);
    ZL_CHECK_ARG(row0 >= 0 && n > 0 && row0 + n <= m->arena.cap[task]);
    ZL_CHECK_ARG(m->cfg.kv_int8 || (!sk_host && !sv_host));
    const Layer& L = m->layers[layer];
    const size_t row = (size_t)m->hkv * m->cfg.dim_head;   // values per token
    const size_t vb = m->cfg.kv_int8 ? 1 : 2;               // bytes per value
    const size_t r0 = (size_t)m->arena.first[task] + row0;
    const size_t off = r0 * row * vb;
    const size_t soff = r0 * m->hkv * 4;
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

// ------------------------------------------------------------------------------------------------------------------
// Prompt prefix cache: the block pool and the block copies (PrefixCache, src/generator/prefix_cache.hpp:35-117).  Which
// blocks to save and load is the caller's policy (zhilight_b200/prefix_cache.py); this owns the memory and the copies.
// ------------------------------------------------------------------------------------------------------------------
extern "C" int zl_llama_kv_pool_create(zl_llama_t* m, int num_blocks, int block_tokens) {
    ZL_CHECK_ARG(m && num_blocks > 0);
    ZL_CHECK_ARG(block_tokens == 16 || block_tokens == 32 || block_tokens == 64 || block_tokens == 128 ||
                 block_tokens == 256);
    if (!m->finalized) return fail_state(__LINE__, "zl_llama_kv_pool_create needs a finalized model");
    if (m->pool) return fail_state(__LINE__, "the KV block pool already exists");
    const auto& c = m->cfg;
    const int L = c.num_layers;
    const int row_bytes = m->hkv * c.dim_head * (c.kv_int8 ? 1 : 2);
    const int srow_bytes = c.kv_int8 ? m->hkv * 4 : 0;
    if (!kv_block_copy_aligned(block_tokens, m->arena.unit(), row_bytes, srow_bytes))
        return fail_state(__LINE__, "KV block copies need max_seq * (bytes of one cached row) to be a multiple of 16",
                          ZL_ERR_UNSUPPORTED);
    const size_t blk = (size_t)block_tokens * row_bytes, sblk = (size_t)block_tokens * srow_bytes;
    const int cap = num_blocks > c.max_seq / block_tokens ? num_blocks : c.max_seq / block_tokens;
    dev_ptr<> pool, scales;
    RCHECK(dmalloc(&pool, (size_t)L * 2 * num_blocks * blk));
    if (c.kv_int8) RCHECK(dmalloc(&scales, (size_t)L * 2 * num_blocks * sblk));
    RCHECK(m->pool_ring.alloc((size_t)2 * cap, true));
    m->pool = std::move(pool);
    m->pool_scales = std::move(scales);
    m->pool_blocks = num_blocks;
    m->pool_bt = block_tokens;
    m->pool_cap = cap;
    return ZL_OK;
}

namespace {

// every check of a save / load before anything is enqueued
int check_kv_blocks(zl_llama* m, int task, const int32_t* task_blocks, const int32_t* pool_blocks, int n, bool to_pool) {
    ZL_CHECK_ARG(m && task_blocks && pool_blocks && n > 0);
    if (!m->finalized || !m->pool) return fail_state(__LINE__, "no KV block pool (zl_llama_kv_pool_create)");
    const auto& c = m->cfg;
    ZL_CHECK_ARG(task >= 0 && task < c.max_batch && n <= m->pool_cap);
    const int task_max = c.max_seq / m->pool_bt;   // (j + 1) * bt <= max_seq
    std::vector<char> seen(to_pool ? m->pool_blocks : task_max, 0);
    for (int i = 0; i < n; ++i) {
        ZL_CHECK_ARG(task_blocks[i] >= 0 && task_blocks[i] < task_max);
        ZL_CHECK_ARG(pool_blocks[i] >= 0 && pool_blocks[i] < m->pool_blocks);
        const int dst = to_pool ? pool_blocks[i] : task_blocks[i];
        ZL_CHECK_ARG(!seen[dst]);   // no destination twice
        seen[dst] = 1;
    }
    return ZL_OK;
}

KvBlockCopyArgs kv_copy_args(zl_llama* m, int task, const int32_t* d_pairs, int n, bool to_pool) {
    const auto& c = m->cfg;
    KvBlockCopyArgs a{};
    a.task_tabs = reinterpret_cast<void* const* const*>(m->kv_tabs.get());
    a.pool = static_cast<char*>(m->pool.get());
    a.pool_scales = static_cast<char*>(m->pool_scales.get());
    a.pairs = d_pairs;
    a.n = n;
    a.layers = c.num_layers;
    a.num_blocks = m->pool_blocks;
    a.bt = m->pool_bt;
    a.task = task;
    a.row_bytes = m->hkv * c.dim_head * (c.kv_int8 ? 1 : 2);
    a.srow_bytes = c.kv_int8 ? m->hkv * 4 : 0;
    a.to_pool = to_pool ? 1 : 0;
    return a;
}

// stage the block lists in the next pool_ring slot -> its device copy; release the slot after the kernel that reads it
int stage_kv_blocks(zl_llama* m, const int32_t* task_blocks, const int32_t* pool_blocks, int n, const int32_t** d_pairs) {
    int32_t *hs = nullptr, *ds = nullptr;
    RCHECK(m->pool_ring.acquire(&hs, &ds));
    std::memcpy(hs, task_blocks, sizeof(int32_t) * n);
    std::memcpy(hs + n, pool_blocks, sizeof(int32_t) * n);
    ZL_CHECK_CUDA(cudaMemcpyAsync(ds, hs, sizeof(int32_t) * 2 * n, cudaMemcpyHostToDevice, m->stream));
    *d_pairs = ds;
    return ZL_OK;
}

// the task's rows the blocks cover, granted before a save reads or a load writes them
int kv_reserve_blocks(zl_llama* m, int task, const int32_t* task_blocks, int n) {
    int rows = 0;
    for (int i = 0; i < n; ++i) rows = std::max(rows, (task_blocks[i] + 1) * m->pool_bt);
    return kv_reserve(m, {{task, rows}});
}

int kv_blocks(zl_llama* m, int task, const int32_t* task_blocks, const int32_t* pool_blocks, int n, bool to_pool) {
    RCHECK(check_kv_blocks(m, task, task_blocks, pool_blocks, n, to_pool));
    RCHECK(kv_reserve_blocks(m, task, task_blocks, n));
    const int32_t* d_pairs = nullptr;
    RCHECK(stage_kv_blocks(m, task_blocks, pool_blocks, n, &d_pairs));
    RCHECK(kv_block_copy(kv_copy_args(m, task, d_pairs, n, to_pool), m->stream));
    return m->pool_ring.release(m->stream);
}

}  // namespace

extern "C" int zl_llama_kv_blocks_save(zl_llama_t* m, int task, const int32_t* task_blocks, const int32_t* pool_blocks,
                                       int n) {
    return kv_blocks(m, task, task_blocks, pool_blocks, n, true);
}

extern "C" int zl_llama_kv_blocks_load(zl_llama_t* m, int task, const int32_t* task_blocks, const int32_t* pool_blocks,
                                       int n) {
    return kv_blocks(m, task, task_blocks, pool_blocks, n, false);
}

extern "C" int zl_llama_kv_blocks_bench(zl_llama_t* m, int task, const int32_t* task_blocks, const int32_t* pool_blocks,
                                        int n, int load, int per_range_memcpy, int iters, float* ms, double* bytes) {
    ZL_CHECK_ARG(iters > 0 && ms);
    const bool to_pool = !load;
    RCHECK(check_kv_blocks(m, task, task_blocks, pool_blocks, n, to_pool));
    RCHECK(kv_reserve_blocks(m, task, task_blocks, n));
    const auto& c = m->cfg;
    const KvBlockCopyArgs a0 = kv_copy_args(m, task, nullptr, 0, to_pool);
    const size_t blk = (size_t)a0.bt * a0.row_bytes, sblk = (size_t)a0.bt * a0.srow_bytes;
    const int32_t* d_pairs = nullptr;
    RCHECK(stage_kv_blocks(m, task_blocks, pool_blocks, n, &d_pairs));
    const KvBlockCopyArgs a = kv_copy_args(m, task, d_pairs, n, to_pool);
    auto one_pass = [&]() -> int {
        if (!per_range_memcpy) return kv_block_copy(a, m->stream);
        for (int i = 0; i < n; ++i)
            for (int l = 0; l < c.num_layers; ++l) {
                const Layer& L = m->layers[l];
                const std::array<void*, 4> tbuf = {L.kbuf.get(), L.vbuf.get(), L.skbuf.get(), L.svbuf.get()};
                for (int t = 0; t < (sblk ? 4 : 2); ++t) {
                    const bool sc = t >= 2;
                    const size_t rb = sc ? a.srow_bytes : a.row_bytes, bb = sc ? sblk : blk;
                    char* tp = static_cast<char*>(tbuf[t]) +
                               ((size_t)m->arena.first[task] + (size_t)task_blocks[i] * a.bt) * rb;
                    char* pp = (sc ? a.pool_scales : a.pool) + ((size_t)(l * 2 + (t & 1)) * a.num_blocks + pool_blocks[i]) * bb;
                    ZL_CHECK_CUDA(cudaMemcpyAsync(to_pool ? pp : tp, to_pool ? tp : pp, bb, cudaMemcpyDeviceToDevice,
                                                  m->stream));
                }
            }
        return ZL_OK;
    };
    cudaEvent_t e0, e1;
    ZL_CHECK_CUDA(cudaEventCreate(&e0));
    ZL_CHECK_CUDA(cudaEventCreate(&e1));
    int rc = one_pass();   // warm-up
    if (rc == ZL_OK) rc = cudaEventRecord(e0, m->stream) == cudaSuccess ? ZL_OK : ZL_ERR_CUDA;
    for (int it = 0; it < iters && rc == ZL_OK; ++it) rc = one_pass();
    if (rc == ZL_OK) rc = cudaEventRecord(e1, m->stream) == cudaSuccess ? ZL_OK : ZL_ERR_CUDA;
    if (rc == ZL_OK) rc = m->pool_ring.release(m->stream);   // after the last pass that reads the device slot
    if (rc == ZL_OK) rc = cudaEventSynchronize(e1) == cudaSuccess ? ZL_OK : ZL_ERR_CUDA;
    if (rc == ZL_OK) rc = cudaEventElapsedTime(ms, e0, e1) == cudaSuccess ? ZL_OK : ZL_ERR_CUDA;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (rc == ZL_ERR_CUDA) zl_set_last_error(__FILE__, __LINE__, "CUDA event failed in zl_llama_kv_blocks_bench");
    if (bytes) *bytes = 2.0 * n * c.num_layers * 2 * (double)(blk + sblk);   // read + write
    return rc;
}

// ------------------------------------------------------------------------------------------------------------------
// Beam search (SearcherImplV1 with beam_size > 1, src/generator/batch_generator.cpp:1762-1852): the decode step with the
// pick replaced by zl_beam_topk, and beam forks as KV row copies between task slots.  The policy -- which candidates live,
// finish or stop a group, and which slot each beam takes -- is the caller's (zhilight_b200/beam_search.py).
// ------------------------------------------------------------------------------------------------------------------
namespace {

constexpr int kBeamK = 32;   // zl_beam_topk's largest K

int ensure_beam(zl_llama* m) {
    if (m->beam_d) return ZL_OK;
    const int MB = m->cfg.max_batch;
    size_t ws = 0;   // the workspace of the largest R <= max_batch
    for (int r = 1; r <= MB; ++r) {
        const size_t b = zl_beam_topk_workspace_bytes(r, m->cfg.vocab_size, kBeamK);
        if (b > ws) ws = b;
    }
    const size_t words = (size_t)MB * (3 + 3 * kBeamK);
    dev_ptr<> d, w;
    RCHECK(dmalloc(&d, words * 4));
    RCHECK(dmalloc(&w, ws));
    int32_t* h = nullptr;
    ZL_CHECK_CUDA(cudaMallocHost((void**)&h, words * 4));
    m->beam_h.reset(h);
    m->beam_d = std::move(d);
    m->beam_ws = std::move(w);
    return ZL_OK;
}

}  // namespace

extern "C" int zl_llama_beam_step(zl_llama_t* m, const int32_t* tokens, const int32_t* positions, int B,
                                  const int32_t* groups, int G, const float* cum, int K, int32_t* parent, int32_t* token,
                                  float* score, float* logits_host) {
    ZL_CHECK_ARG(m && tokens && positions && groups && cum && parent && token && score);
    ZL_CHECK_ARG(B > 0 && B <= m->cfg.max_batch);
    RCHECK(beam_topk_check(B, full_rows(m) ? m->cfg.vocab_size : m->vshard, groups, G, K));
    for (int i = 0; i < B; ++i) ZL_CHECK_ARG(cum[i] < INFINITY);   // -inf: a dead row; NaN and +inf are refused
    RCHECK(need_full_rows(m, "zl_llama_beam_step"));
    ZL_CHECK_SUPPORTED(B < 2048);   // the graph key holds B and G in 11 bits
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    if (pick_of(m, 0, B).sampler)
        return fail_state(__LINE__, "a task of the beam step samples, has penalties, logits processors or a constraint");
    RCHECK(check_state(m, tokens, positions, B));
    RCHECK(ensure_beam(m));
    RCHECK(kv_reserve_step(m, positions, B));
    const int MB = m->cfg.max_batch;
    int32_t* d = static_cast<int32_t*>(m->beam_d.get());
    int32_t* h = m->beam_h.get();
    // layout (max_batch words each, the outputs 32 x max_batch): cum | groups (2) | parent | token | score
    BeamPick bp;
    bp.cum = reinterpret_cast<const float*>(d);
    bp.groups = d + MB;
    bp.G = G;
    bp.K = K;
    bp.parent = d + 3 * MB;
    bp.token = bp.parent + kBeamK * MB;
    bp.score = reinterpret_cast<float*>(bp.token + kBeamK * MB);
    bp.ws = m->beam_ws.get();
    RCHECK(zl_llama_set_state(m, tokens, positions, B));
    std::memcpy(h, cum, sizeof(float) * B);
    std::memcpy(h + MB, groups, sizeof(int32_t) * 2 * G);
    cudaStream_t st = m->stream;
    ZL_CHECK_CUDA(cudaMemcpyAsync(d, h, sizeof(float) * B, cudaMemcpyHostToDevice, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(d + MB, h + MB, sizeof(int32_t) * 2 * G, cudaMemcpyHostToDevice, st));
    RCHECK(run_step(m, B, &bp));
    const size_t n = (size_t)G * K;
    int32_t* hp = h + 3 * MB;
    int32_t* ht = hp + kBeamK * MB;
    int32_t* hs = ht + kBeamK * MB;
    ZL_CHECK_CUDA(cudaMemcpyAsync(hp, bp.parent, n * 4, cudaMemcpyDeviceToHost, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(ht, bp.token, n * 4, cudaMemcpyDeviceToHost, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(hs, bp.score, n * 4, cudaMemcpyDeviceToHost, st));
    if (logits_host)
        ZL_CHECK_CUDA(cudaMemcpyAsync(logits_host, m->logits.get(), (size_t)B * m->vshard * 4, cudaMemcpyDeviceToHost, st));
    ZL_CHECK_CUDA(cudaStreamSynchronize(st));   // also frees the pinned staging for the next call
    std::memcpy(parent, hp, n * 4);
    std::memcpy(token, ht, n * 4);
    std::memcpy(score, hs, n * 4);
    return ZL_OK;
}

extern "C" int zl_llama_kv_copy_rows(zl_llama_t* m, const int32_t* ranges_host, int n) {
    ZL_CHECK_ARG(m && ranges_host && n > 0);
    const auto& c = m->cfg;
    ZL_CHECK_ARG(n <= c.max_batch);
    // every check before anything is enqueued
    std::vector<char> role(c.max_batch, 0);   // 1 source, 2 destination
    int max_rows = 0;
    for (int i = 0; i < n; ++i) {
        const int32_t* r4 = ranges_host + 4 * i;
        ZL_CHECK_ARG(r4[0] >= 0 && r4[0] < c.max_batch && r4[1] >= 0 && r4[1] < c.max_batch && r4[0] != r4[1]);
        ZL_CHECK_ARG(r4[2] >= 0 && r4[2] < r4[3] && r4[3] <= c.max_seq);
        ZL_CHECK_ARG(role[r4[0]] != 2 && role[r4[1]] == 0);   // no destination twice, no task both source and destination
        role[r4[0]] = 1;
        role[r4[1]] = 2;
        if (r4[3] - r4[2] > max_rows) max_rows = r4[3] - r4[2];
    }
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    const int row_bytes = m->hkv * c.dim_head * (c.kv_int8 ? 1 : 2);
    if (row_bytes % 16 != 0)
        return fail_state(__LINE__, "KV row copies need 16-byte cached rows (H_kv * dim_head)", ZL_ERR_UNSUPPORTED);
    // the sources' rows are granted too: the copy reads them through the same tables
    std::vector<std::pair<int, int>> needs;
    for (int i = 0; i < n; ++i)
        for (int t : {ranges_host[4 * i], ranges_host[4 * i + 1]}) needs.push_back({t, ranges_host[4 * i + 3]});
    RCHECK(kv_reserve(m, needs));
    if (!m->rows_ring.h) RCHECK(m->rows_ring.alloc((size_t)4 * c.max_batch, true));
    int32_t *hs = nullptr, *ds = nullptr;
    RCHECK(m->rows_ring.acquire(&hs, &ds));
    std::memcpy(hs, ranges_host, sizeof(int32_t) * 4 * n);
    ZL_CHECK_CUDA(cudaMemcpyAsync(ds, hs, sizeof(int32_t) * 4 * n, cudaMemcpyHostToDevice, m->stream));
    KvRowCopyArgs a{};
    a.task_tabs = reinterpret_cast<void* const* const*>(m->kv_tabs.get());
    a.ranges = ds;
    a.n = n;
    a.layers = c.num_layers;
    a.max_rows = max_rows;
    a.row_bytes = row_bytes;
    a.srow_bytes = c.kv_int8 ? m->hkv * 4 : 0;
    RCHECK(kv_row_copy(a, m->stream));
    return m->rows_ring.release(m->stream);
}

// ------------------------------------------------------------------------------------------------------------------
// Generate until stop (the reference's stop rules, src/generator/batch_generator.cpp:1744-1753, 1812-1817): decode steps
// in a CUDA-graph while loop that applies each task's stop ids, token budget and the end of its KV buffer on the device.
// Graph: k_gen_head -> while (live tasks and steps left) { the decode step; k_gen_advance } -> k_gen_tail.
// ------------------------------------------------------------------------------------------------------------------
namespace {

constexpr int kGenThreads = 256;

struct StopRule {
    int32_t ids[ZL_MAX_STOP_IDS];
    int32_t n, budget;
};

// zl_llama_set_stop: the task's rule, emitted count 0, running
__global__ void k_gen_arm(GenState g, int task, StopRule r) {
    for (int j = 0; j < ZL_MAX_STOP_IDS; ++j) g.stop[task * ZL_MAX_STOP_IDS + j] = r.ids[j];
    g.n_stop[task] = r.n;
    g.budget[task] = r.budget;
    g.emitted[task] = 0;
    g.fin[task] = 0;
}

// before each graph launch of a call: the step counter (first launch) and the steps this launch may run
__global__ void k_gen_begin(GenState g, int first, int steps) {
    if (first) g.ctl[0] = 0;
    g.ctl[1] = steps;
}

__device__ int gen_block_sum(int v) {
    __shared__ int part[kGenThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    int s = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kGenThreads / 32; ++w) s += part[w];
    return s;   // thread 0
}

// A task whose state position is max_seq (it stopped at max_seq - 1) cannot be fed there: while the launch runs it
// re-feeds its last (token, position), which rewrites that KV row with what it already holds.  A task re-armed in that
// state finishes at once (reason 3) without emitting.  Then the loop's first condition: running tasks and steps left.
__global__ void __launch_bounds__(kGenThreads) k_gen_head(GenState g, int32_t* __restrict__ tokens,
                                                          int32_t* __restrict__ pos, int B, cudaGraphConditionalHandle h) {
    int live = 0;
    for (int i = threadIdx.x; i < B; i += kGenThreads) {
        if (pos[i] >= g.max_seq) {
            g.stok[i] = tokens[i];
            tokens[i] = g.ftok[i];
            pos[i] = g.max_seq - 1;
            g.edge[i] = 1;
            if (g.fin[i] == 0) g.fin[i] = 3;
        }
        live += g.fin[i] == 0;
    }
    live = gen_block_sum(live);
    if (threadIdx.x == 0) cudaGraphSetConditional(h, live > 0 && g.ctl[1] > 0);
}

// In place of k_advance: each running task emits its pick into ring row `step`, applies its stop rules and is fed its
// pick at the next position; a finished task's row emits -1 and keeps its state.  Sets the loop condition.
__global__ void __launch_bounds__(kGenThreads) k_gen_advance(GenState g, int32_t* __restrict__ tokens,
                                                             int32_t* __restrict__ pos, const int32_t* __restrict__ next,
                                                             int B, cudaGraphConditionalHandle h) {
    const int step = g.ctl[0];
    int live = 0;
    for (int i = threadIdx.x; i < B; i += kGenThreads) {
        int out = -1;
        if (g.fin[i] == 0) {
            const int tok = next[i];
            out = tok;
            const int e = g.emitted[i] + 1;
            g.emitted[i] = e;
            const int p1 = pos[i] + 1;
            int reason = 0;
            for (int j = 0; j < g.n_stop[i]; ++j)
                if (g.stop[i * ZL_MAX_STOP_IDS + j] == tok) reason = 1;
            if (!reason && g.budget[i] > 0 && e >= g.budget[i]) reason = 2;
            if (!reason && p1 >= g.max_seq) reason = 3;
            if (p1 < g.max_seq) {
                tokens[i] = tok;
                pos[i] = p1;
            } else {   // the buffer is full: the state (tok, max_seq) is restored by k_gen_tail
                g.ftok[i] = tokens[i];
                g.stok[i] = tok;
                g.edge[i] = 1;
            }
            g.fin[i] = reason;
            live += reason == 0;
        }
        g.ring[(size_t)step * g.max_batch + i] = out;
    }
    live = gen_block_sum(live);
    if (threadIdx.x == 0) {
        const int left = g.ctl[1] - 1;
        g.ctl[0] = step + 1;
        g.ctl[1] = left;
        cudaGraphSetConditional(h, live > 0 && left > 0);
    }
}

// after the loop: the tasks that re-fed max_seq - 1 get back their state (emitted token, max_seq)
__global__ void k_gen_tail(GenState g, int32_t* __restrict__ tokens, int32_t* __restrict__ pos, int B) {
    for (int i = threadIdx.x; i < B; i += blockDim.x)
        if (g.edge[i]) {
            tokens[i] = g.stok[i];
            pos[i] = g.max_seq;
            g.edge[i] = 0;
        }
}

// The loop graph of (B, pick, bucket) into *out, which the caller owns also when this fails.  The body keeps the step's
// programmatic dependent launches.
int build_gen_graph(zl_llama* m, int B, const Pick& pk, int bucket, cudaGraph_t* out) {
    GenState gs = gen_state(m);
    int32_t* tokens = m->d_tokens.get();
    int32_t* pos = m->d_pos.get();
    const int32_t* next = m->d_next.get();
    ZL_CHECK_CUDA(cudaGraphCreate(out, 0));
    cudaGraph_t g = *out;
    cudaGraphConditionalHandle h;
    ZL_CHECK_CUDA(cudaGraphConditionalHandleCreate(&h, g, 0, 0));
    cudaKernelNodeParams kp = {};
    void* head_args[] = {&gs, &tokens, &pos, &B, &h};
    kp.func = (void*)k_gen_head;
    kp.gridDim = dim3(1);
    kp.blockDim = dim3(kGenThreads);
    kp.kernelParams = head_args;
    cudaGraphNode_t head = nullptr, loop = nullptr, tail = nullptr;
    ZL_CHECK_CUDA(cudaGraphAddKernelNode(&head, g, nullptr, 0, &kp));
    cudaGraphNodeParams cp = {};
    cp.type = cudaGraphNodeTypeConditional;
    cp.conditional.handle = h;
    cp.conditional.type = cudaGraphCondTypeWhile;
    cp.conditional.size = 1;
    ZL_CHECK_CUDA(cudaGraphAddNode(&loop, g, &head, 1, &cp));
    cudaGraph_t body = cp.conditional.phGraph_out[0];
    // the body: the unchanged decode step, then k_gen_advance in k_advance's place
    ZL_CHECK_CUDA(cudaStreamBeginCaptureToGraph(m->stream, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    Pick body_pick = pk;
    body_pick.frozen = gs.fin;   // the sampler records no pick of a finished task
    int rc = enqueue_step(m, B, bucket, nullptr, body_pick);
    if (rc == ZL_OK) {
        k_gen_advance<<<1, kGenThreads, 0, m->stream>>>(gs, tokens, pos, next, B, h);
        if (cudaGetLastError() != cudaSuccess) rc = fail_state(__LINE__, "k_gen_advance launch failed", ZL_ERR_CUDA);
    }
    const cudaError_t ce = cudaStreamEndCapture(m->stream, &body);
    if (rc != ZL_OK) return rc;
    ZL_CHECK_CUDA(ce);
    void* tail_args[] = {&gs, &tokens, &pos, &B};
    kp.func = (void*)k_gen_tail;
    kp.kernelParams = tail_args;
    ZL_CHECK_CUDA(cudaGraphAddKernelNode(&tail, g, &loop, 1, &kp));
    return ZL_OK;
}

}  // namespace

extern "C" int zl_llama_set_stop(zl_llama_t* m, int task, const int32_t* stop_ids_host, int n_stop, int max_new_tokens) {
    ZL_CHECK_ARG(m && task >= 0 && task < m->cfg.max_batch);
    ZL_CHECK_ARG(n_stop >= 0 && n_stop <= ZL_MAX_STOP_IDS && (n_stop == 0 || stop_ids_host));
    ZL_CHECK_ARG(max_new_tokens >= 0);
    StopRule r{};
    for (int j = 0; j < n_stop; ++j) {
        ZL_CHECK_ARG(stop_ids_host[j] >= 0 && stop_ids_host[j] < m->cfg.vocab_size);
        for (int k = 0; k < j; ++k) ZL_CHECK_ARG(stop_ids_host[k] != stop_ids_host[j]);
        r.ids[j] = stop_ids_host[j];
    }
    r.n = n_stop;
    r.budget = max_new_tokens;
    RCHECK(need_full_rows(m, "zl_llama_set_stop"));
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    // stream-ordered after every step already enqueued; the rule travels as a kernel argument
    k_gen_arm<<<1, 1, 0, m->stream>>>(gen_state(m), task, r);
    ZL_CHECK_LAUNCH();
    m->gen_fin[task] = 0;
    return ZL_OK;
}

extern "C" int zl_llama_generate(zl_llama_t* m, int B, int max_steps, int32_t* tokens_host, int32_t* n_out_host,
                                 int32_t* finish_host, int* steps_host) {
    ZL_CHECK_ARG(m && tokens_host && n_out_host && finish_host && steps_host);
    const auto& c = m->cfg;
    ZL_CHECK_ARG(B > 0 && B <= c.max_batch && max_steps >= 1 && max_steps <= c.max_seq);
    RCHECK(need_full_rows(m, "zl_llama_generate"));
    if (!c.use_graph) return fail_state(__LINE__, "zl_llama_generate runs as a CUDA graph (use_graph = 0)", ZL_ERR_UNSUPPORTED);
    if (!m->finalized) return fail_state(__LINE__, "model not finalized");
    const int MB = c.max_batch;
    bool all_done = true;
    for (int i = 0; i < B; ++i) all_done = all_done && m->gen_fin[i] != 0;
    if (all_done) {
        for (size_t k = 0; k < (size_t)max_steps * B; ++k) tokens_host[k] = -1;
        for (int i = 0; i < B; ++i) {
            n_out_host[i] = 0;
            finish_host[i] = m->gen_fin[i];
        }
        *steps_host = 0;
        return ZL_OK;
    }
    // every row the call can write: min(pos + max_steps, max_seq) rows of a running task; a finished task re-runs its
    // state position (max_seq - 1 at the end of its buffer)
    std::vector<std::pair<int, int>> needs(B);
    for (int i = 0; i < B; ++i)
        needs[i] = {i, std::min(m->pos_host[i] + (m->gen_fin[i] ? 1 : max_steps), c.max_seq)};
    RCHECK(kv_reserve(m, needs));
    const Pick pk = pick_of(m, 0, B);
    const GenState gs = gen_state(m);
    // attention lengths at step s are at most min(L0 + s, max_seq): one launch per length bucket crossed
    const int L0 = m->cur_max_len;
    for (int s = 0; s < max_steps;) {
        const int len = std::min(L0 + s, c.max_seq);
        const int bucket = len_bucket_of(m, len);
        int n = max_steps - s;
        if (bucket < c.max_seq) n = std::min(n, bucket - (L0 + s) + 1);
        cudaGraphExec_t exec = nullptr;
        RCHECK(m->gen_graphs.get(
            graph_key(B, pk, bucket),
            [&](cudaGraph_t* g) { return build_gen_graph(m, B, pk, bucket, g); }, &exec));
        k_gen_begin<<<1, 1, 0, m->stream>>>(gs, s == 0, n);
        ZL_CHECK_LAUNCH();
        ZL_CHECK_CUDA(cudaGraphLaunch(exec, m->stream));
        s += n;
    }
    // one sync: ring rows | finish reasons | positions | control
    int32_t* h_ring = m->h_gen.get();
    int32_t* h_fin = h_ring + (size_t)c.max_seq * MB;
    int32_t* h_pos = h_fin + MB;
    int32_t* h_ctl = h_pos + MB;
    cudaStream_t st = m->stream;
    ZL_CHECK_CUDA(cudaMemcpyAsync(h_ring, gs.ring, (size_t)max_steps * MB * 4, cudaMemcpyDeviceToHost, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(h_fin, gs.fin, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(h_pos, m->d_pos.get(), (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    ZL_CHECK_CUDA(cudaMemcpyAsync(h_ctl, gs.ctl, kGenCtlWords * 4, cudaMemcpyDeviceToHost, st));
    ZL_CHECK_CUDA(cudaStreamSynchronize(st));
    const int steps = h_ctl[0];
    for (int i = 0; i < B; ++i) n_out_host[i] = 0;
    for (int s = 0; s < max_steps; ++s)
        for (int i = 0; i < B; ++i) {
            const int32_t t = s < steps ? h_ring[(size_t)s * MB + i] : -1;
            tokens_host[(size_t)s * B + i] = t;
            n_out_host[i] += t >= 0;
        }
    int mx = m->cur_max_len;
    for (int i = 0; i < B; ++i) {
        finish_host[i] = h_fin[i];
        m->gen_fin[i] = (char)h_fin[i];
        m->pos_host[i] = h_pos[i];
        mx = std::max(mx, h_pos[i] + 1);
    }
    m->cur_max_len = mx;
    *steps_host = steps;
    return ZL_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// KV arena (cfg.kv_rows > 0): each task's rows come from one shared row space as its writes reach them (KvArena).
// ------------------------------------------------------------------------------------------------------------------
extern "C" int zl_llama_kv_release(zl_llama_t* m, int task) {
    ZL_CHECK_ARG(m && task >= 0 && task < m->cfg.max_batch);
    m->arena.release(task);
    return ZL_OK;
}

extern "C" int zl_llama_kv_capacity(zl_llama_t* m, int task, int* rows) {
    ZL_CHECK_ARG(m && rows && task >= 0 && task < m->cfg.max_batch);
    *rows = m->arena.cap[task];
    return ZL_OK;
}

extern "C" int zl_llama_kv_free_rows(zl_llama_t* m, int* rows) {
    ZL_CHECK_ARG(m && rows);
    *rows = m->arena.free_rows();
    return ZL_OK;
}
