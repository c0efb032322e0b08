// TEST INFRASTRUCTURE (oracle/_ref): a thin extern "C" shim over the REFERENCE's own hot-path kernels.
//
// Built by oracle/Makefile.ref from the sources where they lie in a reference checkout (never copied into
// this repo) into oracle/_ref/libzl_ref.so.  It lets the GPU parity tests and oracle/gen_ref_golden.py run
// the reference's kernels (recompiled for sm_90a) on the same device buffers as ours.  Only tests/,
// __graft_entry__ and bench tooling may load it; the product library never links or dlopens it.
//
// All pointers are device pointers; every call runs on the shim's private bmengine Context/stream and
// synchronises before returning (this is a checker, not a fast path).
#include <bmengine/core/core.h>
#include <bmengine/functions/transpose.h>

#include "nn/quant/gptq/gptq.h"
#include "nn/quant/int8/quant_kernel.h"
#include "nn/quant/fp8/fp8.h"
#include <bmengine/functions/gemm.h>
#include "nn/attention/attention_kernel.h"
#include "nn/layernorm/layernorm.h"
#include "nn/position/rotary_embedding.h"
#include "nn/block/block_kernel.h"
#include "nn/linear/activation_kernel.h"
#include "kvcache/ragged_buffer_kernel.h"
#include "nn/position/rope_preparer.h"

#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>

using namespace bmengine;
using core::DataType;
using core::Tensor;

// gptq_gemm_k_major does dynamic_cast<model::ModelContext*>(ctx) (q_gemm_k_major.cu:994); only the typeinfo
// symbol is needed at link time.  A plain core::Context is never a ModelContext, so the cast yields nullptr,
// which is the code path a standalone Linear test takes.
namespace model {
class ModelContext {
public:
    virtual ~ModelContext();
};
ModelContext::~ModelContext() {}
}  // namespace model

namespace {
std::unique_ptr<core::Engine> g_engine;
std::unique_ptr<core::Context> g_ctx;
std::unique_ptr<core::WithDevice> g_dev;
char g_err[1024] = "";

Tensor wrap(std::vector<size_t> shape, DataType dt, const void* p) {
    size_t n = 1;
    for (auto s : shape) n *= s;
    return Tensor::from_external(shape, dt, const_cast<void*>(p), n * core::get_elem_size(dt), 0, false);
}
DataType dt_of(int code) { return code == 1 ? DataType::kBFloat16 : (code == 2 ? DataType::kFloat : DataType::kHalf); }
void sync() { BM_CUDART_ASSERT(cudaStreamSynchronize(g_ctx->current_stream()->ptr)); }
void copy_out(const Tensor& t, void* dst) {
    BM_CUDART_ASSERT(cudaMemcpyAsync(dst, t.data(), t.nbytes(), cudaMemcpyDeviceToDevice, g_ctx->current_stream()->ptr));
}
}  // namespace

// accessors for ref_shim_r2.cu
core::Context* zlref_ctx() { return g_ctx.get(); }
char* zlref_err_buf() { return g_err; }

#define ZLREF_TRY(...)                                         \
    try {                                                      \
        __VA_ARGS__;                                           \
        sync();                                                \
        return 0;                                              \
    } catch (const std::exception& e) {                        \
        snprintf(g_err, sizeof(g_err), "%s", e.what());        \
        return -1;                                             \
    }

extern "C" {

const char* zlref_last_error() { return g_err; }

int zlref_init(int device, size_t mem_bytes) {
    try {
        if (g_ctx) return 0;
        std::vector<core::DeviceConfiguration> devs;
        devs.emplace_back(device, mem_bytes);
        g_engine.reset(new core::Engine(devs));
        g_ctx.reset(new core::Context(g_engine->create_context({0})));
        g_dev.reset(new core::WithDevice(g_ctx->with_device(0)));
        g_ctx->set_BSHD(true);
        return 0;
    } catch (const std::exception& e) {
        snprintf(g_err, sizeof(g_err), "%s", e.what());
        return -1;
    }
}

// ---- load-time layout transforms (in place unless an out pointer is given) ----
int zlref_gptq_shuffle(void* qweight, int K, int N) {
    ZLREF_TRY(Tensor w = wrap({(size_t)K / 8, (size_t)N}, DataType::kInt32, qweight);
              nn::gptq::gptq_shuffle(*g_ctx, w, Tensor()))
}
int zlref_increase_zero(void* qzeros, int rows, int cols) {
    ZLREF_TRY(Tensor z = wrap({(size_t)rows, (size_t)cols}, DataType::kInt32, qzeros);
              nn::gptq::increase_zero(*g_ctx, z))
}
int zlref_q4_to_q8(const void* in, int rows, int cols, void* out) {
    ZLREF_TRY(Tensor z = wrap({(size_t)rows, (size_t)cols}, DataType::kInt32, in);
              Tensor o = nn::gptq::q4_to_q8(*g_ctx, z); copy_out(o, out))
}
int zlref_un_shuffle(void* qzeros, int rows, int cols) {
    ZLREF_TRY(Tensor z = wrap({(size_t)rows, (size_t)cols}, DataType::kInt32, qzeros);
              nn::gptq::un_shuffle(*g_ctx, z))
}
int zlref_shuffle_awq(const void* in, int K, int N, int use_exllama, void* out) {
    ZLREF_TRY(Tensor w = wrap({(size_t)K, (size_t)N / 8}, DataType::kInt32, in);
              Tensor o = nn::gptq::shuffle_awq(*g_ctx, w, use_exllama != 0); copy_out(o, out))
}
int zlref_transpose(const void* in, int rows, int cols, int elem_bytes, void* out) {
    ZLREF_TRY(DataType dt = elem_bytes == 4 ? DataType::kInt32 : (elem_bytes == 2 ? DataType::kHalf : DataType::kInt8);
              Tensor x = wrap({(size_t)rows, (size_t)cols}, dt, in); functions::Transpose tr(*g_ctx);
              Tensor o = tr(*g_ctx, x); copy_out(o, out))
}
int zlref_dequant_k_major(const void* qw, const void* qz, const void* sc, int N, int K, int G, void* out_f16) {
    ZLREF_TRY(Tensor w = wrap({(size_t)N, (size_t)K / 8}, DataType::kInt32, qw);
              Tensor z = wrap({(size_t)N, (size_t)G}, DataType::kInt8, qz);
              Tensor s = wrap({(size_t)N, (size_t)G}, DataType::kHalf, sc);
              Tensor o = nn::gptq::dequant_k_major(*g_ctx, w, z, s, 0); copy_out(o, out_f16))
}

// ---- W4A16 GEMV (the reference's default decode kernel) ----
int zlref_gptq_gemm_k_major(const void* a, const void* qw, const void* qz, const void* sc, const void* bias, int sym,
                            int M, int N, int K, int G, void* out) {
    ZLREF_TRY(Tensor A = wrap({(size_t)M, (size_t)K}, DataType::kHalf, a);
              Tensor w = wrap({(size_t)N, (size_t)K / 8}, DataType::kInt32, qw); w.set_name("zlref.linear");
              Tensor z = wrap({(size_t)N, (size_t)G}, DataType::kInt8, qz);
              Tensor s = wrap({(size_t)N, (size_t)G}, DataType::kHalf, sc);
              Tensor b = bias ? wrap({(size_t)N}, DataType::kHalf, bias) : Tensor();
              Tensor o = wrap({(size_t)M, (size_t)N}, DataType::kHalf, out);
              nn::gptq::gptq_gemm_k_major(*g_ctx, A, w, z, s, Tensor(), Tensor(), bias ? &b : nullptr, sym != 0, false, &o))
}
int zlref_gemm_fuse_gate_in(const void* a, const void* qw1, const void* qz1, const void* sc1, const void* qw2,
                            const void* qz2, const void* sc2, int sym, int M, int N, int K, int G, void* out) {
    ZLREF_TRY(Tensor A = wrap({(size_t)M, (size_t)K}, DataType::kHalf, a);
              Tensor w1 = wrap({(size_t)N, (size_t)K / 8}, DataType::kInt32, qw1);
              Tensor z1 = wrap({(size_t)N, (size_t)G}, DataType::kInt8, qz1);
              Tensor s1 = wrap({(size_t)N, (size_t)G}, DataType::kHalf, sc1);
              Tensor w2 = wrap({(size_t)N, (size_t)K / 8}, DataType::kInt32, qw2);
              Tensor z2 = wrap({(size_t)N, (size_t)G}, DataType::kInt8, qz2);
              Tensor s2 = wrap({(size_t)N, (size_t)G}, DataType::kHalf, sc2);
              Tensor o = nn::gptq::gemm_fuse_gate_in(*g_ctx, A, w1, z1, s1, Tensor(), w2, z2, s2, Tensor(), sym != 0);
              copy_out(o, out))
}

// ---- norm / residual / activation ----
int zlref_rmsnorm(const void* x, const void* w, int T, int D, float eps, int dtype, void* out) {
    ZLREF_TRY(DataType dt = dt_of(dtype); nn::LayerNorm ln(*g_ctx, D, false, eps, 1.0f, dt);
              std::map<std::string, const Tensor> sd; sd.emplace("ln.weight", wrap({(size_t)D}, dt, w));
              ln.load_state_dict(*g_ctx, sd, "ln", false);
              Tensor X = wrap({(size_t)T, (size_t)D}, dt, x); Tensor o = ln.forward(*g_ctx, X); copy_out(o, out))
}
int zlref_rmsnorm_fuse_add(const void* a, const void* b, const void* w, int T, int D, float eps, int dtype,
                           void* out_sum, void* out) {
    ZLREF_TRY(DataType dt = dt_of(dtype); nn::LayerNorm ln(*g_ctx, D, false, eps, 1.0f, dt);
              std::map<std::string, const Tensor> sd; sd.emplace("ln.weight", wrap({(size_t)D}, dt, w));
              ln.load_state_dict(*g_ctx, sd, "ln", false);
              Tensor A = wrap({(size_t)T, (size_t)D}, dt, a); Tensor B = wrap({(size_t)T, (size_t)D}, dt, b);
              Tensor S = wrap({(size_t)T, (size_t)D}, dt, out_sum); Tensor o = ln.fuse_add(*g_ctx, A, B, S);
              copy_out(o, out))
}
int zlref_element_add_scale(const void* a, const void* b, size_t n, float scale, int dtype, void* out) {
    ZLREF_TRY(DataType dt = dt_of(dtype); Tensor A = wrap({n}, dt, a); Tensor B = wrap({n}, dt, b);
              Tensor C = wrap({n}, dt, out); nn::element_add_scale_out(*g_ctx, A, B, C, scale, false))
}
int zlref_gate_mul_inplace(void* gate, const void* up, int T, int F, int dtype) {
    ZLREF_TRY(DataType dt = dt_of(dtype); Tensor G = wrap({(size_t)T, (size_t)F}, dt, gate);
              Tensor U = wrap({(size_t)T, (size_t)F}, dt, up); nn::gate_mul_inplace(*g_ctx, G, U, "silu"))
}

// ---- RoPE / KV append / decode attention ----
int zlref_rope_qk_cache(const void* cos, const void* sin, const void* qkv, int T, int hq, int hkv, int d, int dtype,
                        void* q, void* k, void* v) {
    ZLREF_TRY(DataType dt = dt_of(dtype); Tensor C = wrap({(size_t)T, (size_t)d}, DataType::kFloat, cos);
              Tensor S = wrap({(size_t)T, (size_t)d}, DataType::kFloat, sin);
              Tensor I = wrap({(size_t)T, (size_t)(hq + 2 * hkv) * d}, dt, qkv); Tensor oq; Tensor ok; Tensor ov;
              nn::rope_qk_cache(*g_ctx, C, S, I, oq, ok, ov, hq, hkv, d, dt, true);
              copy_out(oq, q); copy_out(ok, k); copy_out(ov, v))
}
int zlref_copy_to_rag_buffer2(const void* placement, const void* buf_lens, const void* k_src, const void* v_src,
                              void* k_addrs, void* v_addrs, int B, int len_q, int hkv, int d, int dtype) {
    ZLREF_TRY(DataType dt = dt_of(dtype); Tensor P = wrap({(size_t)B, (size_t)len_q}, DataType::kInt32, placement);
              Tensor L = wrap({(size_t)B}, DataType::kInt32, buf_lens);
              Tensor K = wrap({(size_t)B, (size_t)len_q, (size_t)hkv, (size_t)d}, dt, k_src);
              Tensor V = wrap({(size_t)B, (size_t)len_q, (size_t)hkv, (size_t)d}, dt, v_src);
              Tensor KA = wrap({(size_t)B}, DataType::kDouble, k_addrs); Tensor VA = wrap({(size_t)B}, DataType::kDouble, v_addrs);
              nn::copy_to_rag_buffer2(*g_ctx, P, L, K, V, &KA, &VA, false))
}
int zlref_mqa_rag_buffer(const void* q, const void* buf_lens, const void* k_addrs, const void* v_addrs, const void* mask,
                         size_t mask_len, float scale, int max_len_buf, int B, int len_q, int hq, int hkv, int d,
                         int dtype, int algo_id, void* out) {
    ZLREF_TRY(DataType dt = dt_of(dtype); Tensor Q = wrap({(size_t)B, (size_t)len_q, (size_t)hq, (size_t)d}, dt, q);
              Tensor L = wrap({(size_t)B}, DataType::kInt32, buf_lens);
              Tensor KA = wrap({(size_t)B}, DataType::kDouble, k_addrs); Tensor VA = wrap({(size_t)B}, DataType::kDouble, v_addrs);
              Tensor M = wrap({mask_len}, DataType::kInt8, mask);
              Tensor O = wrap({(size_t)B, (size_t)len_q, (size_t)hq, (size_t)d}, dt, out);
              nn::multi_query_attention_rag_buffer(*g_ctx, Q, L, KA, VA, M, scale, max_len_buf, O, hq / hkv, algo_id))
}

// ---- INT8 helpers (SmoothQuant act quant, TP all-reduce stages) ----
int zlref_quant_calc_scale(const void* x, int M, int K, int dtype, void* out_q, void* out_scale) {
    ZLREF_TRY(Tensor X = wrap({(size_t)M, (size_t)K}, dt_of(dtype), x); Tensor Qo = wrap({(size_t)M, (size_t)K}, DataType::kInt8, out_q);
              Tensor So = wrap({(size_t)M}, DataType::kFloat, out_scale); int8_op::quant_calc_scale(*g_ctx, X, &Qo, &So))
}
int zlref_quant_scale_back(const void* acc_i32, const void* sx, const void* sy, int sy_dtype, int M, int N, int dtype,
                           void* out) {
    ZLREF_TRY(Tensor A = wrap({(size_t)M, (size_t)N}, DataType::kInt32, acc_i32); Tensor SX = wrap({(size_t)M}, DataType::kFloat, sx);
              Tensor SY = wrap({(size_t)N}, dt_of(sy_dtype), sy); Tensor O = wrap({(size_t)M, (size_t)N}, dt_of(dtype), out);
              int8_op::quant_scale_back(*g_ctx, A, &SX, &SY, dt_of(dtype), &O))
}
int zlref_layernorm_quant(const void* x, const void* w, int T, int D, float eps, float scale, int dtype, void* out,
                          void* out_q, void* out_scale) {
    ZLREF_TRY(DataType dt = dt_of(dtype); Tensor X = wrap({(size_t)T, (size_t)D}, dt, x); Tensor W = wrap({(size_t)D}, dt, w);
              Tensor O = wrap({(size_t)T, (size_t)D}, dt, out); Tensor Q = wrap({(size_t)T, (size_t)D}, DataType::kInt8, out_q);
              Tensor S = wrap({(size_t)T}, DataType::kFloat, out_scale); int8_op::layernorm_quant(*g_ctx, X, W, &O, &Q, &S, eps, scale))
}
int zlref_fp8_dynamic_scaled_quant(const void* x, int M, int K, int dtype, void* out_q, void* out_scale) {
    ZLREF_TRY(Tensor X = wrap({(size_t)M, (size_t)K}, dt_of(dtype), x); Tensor q = nn::fp8::dynamic_scaled_quant(*g_ctx, X);
              copy_out(q, out_q); copy_out(*q.quant_scale, out_scale))
}
// Fp8Linear::forward's GEMM (linear.cpp:1675-1680): functions::Gemm(kFP8_E4M3, transA=false, transB=true) with A/B scales
int zlref_fp8_gemm(const void* xq, const void* sx, const void* wq, const void* sw, const void* bias, int M, int N, int K,
                   int dtype, void* out) {
    // Gemm::impl::gemm wants the activation allocation rounded up to 32 rows (gemm.cpp:287), which is how
    // dynamic_scaled_quant allocates its output (fp8_util.cu:191-192): copy into such a buffer
    ZLREF_TRY(DataType dt = dt_of(dtype);
              Tensor A = g_ctx->tensor({(size_t)M, (size_t)K}, DataType::kFP8_E4M3, "", 32 * (size_t)K);
              BM_CUDART_ASSERT(cudaMemcpyAsync(A.data(), xq, (size_t)M * K, cudaMemcpyDeviceToDevice, g_ctx->current_stream()->ptr));
              Tensor W = wrap({(size_t)N, (size_t)K}, DataType::kFP8_E4M3, wq); Tensor SA = wrap({1}, DataType::kFloat, sx);
              Tensor SB = wrap({1}, DataType::kFloat, sw); Tensor B; if (bias) B = wrap({(size_t)N}, dt, bias);
              functions::Gemm gemm(*g_ctx, DataType::kFP8_E4M3, false, true, 1.f); gemm.set_output_type(dt);
              gemm.set_A_scale(SA); gemm.set_B_scale(SB); Tensor r = gemm.forward(*g_ctx, A, W, nullptr, bias ? &B : nullptr);
              copy_out(r, out))
}
int zlref_quant_group_32(const void* x, size_t M, int dtype, void* out_q, void* out_scale) {
    ZLREF_TRY(Tensor X = wrap({M, 32}, dt_of(dtype), x); auto r = int8_op::quant_group_32(*g_ctx, X);
              copy_out(std::get<0>(r), out_q); copy_out(std::get<1>(r), out_scale))
}
int zlref_dequant_sum_quant_g32(const void* my, const void* q_others, const void* s_others, int WS, size_t M, int dtype,
                                void* out_q, void* out_scale) {
    ZLREF_TRY(DataType dt = dt_of(dtype); Tensor my_t = wrap({M, 32}, dt, my);
              Tensor qo = wrap({(size_t)WS - 1, M, 32}, DataType::kInt8, q_others);
              Tensor so = wrap({(size_t)WS - 1, M}, dt, s_others); Tensor oq = wrap({M, 32}, DataType::kInt8, out_q);
              Tensor os = wrap({M}, dt, out_scale); int8_op::dequant_sum_quant_g32(*g_ctx, my_t, qo, so, &oq, &os))
}
int zlref_dequant_group_32(const void* q, const void* scale, size_t M, int dtype, void* out) {
    ZLREF_TRY(DataType dt = dt_of(dtype); Tensor Q = wrap({M, 32}, DataType::kInt8, q); Tensor S = wrap({M}, dt, scale);
              Tensor O = wrap({M, 32}, dt, out); int8_op::dequant_group_32(*g_ctx, Q, S, &O))
}

// ---- timing helper: average microseconds of `iters` back-to-back reference GEMV calls ----
int zlref_time_gptq_gemv(const void* a, const void* const* qw_list, const void* qz, const void* sc, int n_rot, int sym,
                         int M, int N, int K, int G, void* out, int iters, float* us) {
    try {
        Tensor A = wrap({(size_t)M, (size_t)K}, DataType::kHalf, a);
        Tensor z = wrap({(size_t)N, (size_t)G}, DataType::kInt8, qz);
        Tensor s = wrap({(size_t)N, (size_t)G}, DataType::kHalf, sc);
        Tensor o = wrap({(size_t)M, (size_t)N}, DataType::kHalf, out);
        std::vector<Tensor> ws;
        for (int i = 0; i < n_rot; ++i) {
            ws.push_back(wrap({(size_t)N, (size_t)K / 8}, DataType::kInt32, qw_list[i]));
            ws.back().set_name("zlref.linear");
        }
        auto st = g_ctx->current_stream()->ptr;
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        for (int i = 0; i < 3; ++i)
            nn::gptq::gptq_gemm_k_major(*g_ctx, A, ws[i % n_rot], z, s, Tensor(), Tensor(), nullptr, sym != 0, false, &o);
        cudaEventRecord(e0, st);
        for (int i = 0; i < iters; ++i)
            nn::gptq::gptq_gemm_k_major(*g_ctx, A, ws[i % n_rot], z, s, Tensor(), Tensor(), nullptr, sym != 0, false, &o);
        cudaEventRecord(e1, st);
        cudaEventSynchronize(e1);
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        *us = ms * 1e3f / iters;
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        return 0;
    } catch (const std::exception& e) {
        snprintf(g_err, sizeof(g_err), "%s", e.what());
        return -1;
    }
}

// ---- RopePreparer (src/nn/position/rope_preparer.cu:49-233): cos/sin tables, plain and llama3 ----
int zlref_rope_cos_sin(const void* pos, int T, int d, float theta, int llama3, float factor, float low, float high,
                       int orig_ctx, void* out_cos, void* out_sin) {
    ZLREF_TRY(model::ModelConfig cfg("llama", 1, 64, 1, d, 64, 64); cfg.rope_theta = theta;
              if (llama3) { cfg.rope_cfg.type = "llama3"; cfg.rope_cfg.factor = factor; cfg.rope_cfg.low_freq_factor = low;
                            cfg.rope_cfg.high_freq_factor = high; cfg.rope_cfg.original_max_position = orig_ctx; }
              nn::RopePreparer prep(*g_ctx, cfg); Tensor P = wrap({(size_t)T}, DataType::kInt32, pos);
              auto cs = prep.forward(*g_ctx, P, P); copy_out(std::get<0>(cs), out_cos); copy_out(std::get<1>(cs), out_sin))
}

// ---- int8 KV cache (KV_CACHE_DTYPE=int8): cache-side quantisation and the split-KV quant attention kernel ----
int zlref_quant_calc_scale_u8(const void* x, int M, int K, int dtype, void* out_q, void* out_scale) {
    ZLREF_TRY(Tensor X = wrap({(size_t)M, (size_t)K}, dt_of(dtype), x); Tensor Qo = wrap({(size_t)M, (size_t)K}, DataType::kInt8, out_q);
              Tensor So = wrap({(size_t)M}, DataType::kFloat, out_scale); int8_op::quant_calc_scale(*g_ctx, X, &Qo, &So, 127, 128))
}
int zlref_mqa_rag_buffer_quant(const void* q, const void* buf_lens, const void* k_addrs, const void* v_addrs,
                               const void* sk_addrs, const void* sv_addrs, const void* mask, size_t mask_len, float scale,
                               int max_len_buf, int B, int len_q, int hq, int hkv, int d, int out_dtype, void* out) {
    ZLREF_TRY(Tensor Q = wrap({(size_t)B, (size_t)len_q, (size_t)hq, (size_t)d}, DataType::kHalf, q);
              Tensor L = wrap({(size_t)B}, DataType::kInt32, buf_lens);
              Tensor KA = wrap({(size_t)B}, DataType::kDouble, k_addrs); Tensor VA = wrap({(size_t)B}, DataType::kDouble, v_addrs);
              Tensor SKA = wrap({(size_t)B}, DataType::kDouble, sk_addrs); Tensor SVA = wrap({(size_t)B}, DataType::kDouble, sv_addrs);
              Tensor M = wrap({mask_len}, DataType::kInt8, mask);
              Tensor O = wrap({(size_t)B, (size_t)len_q, (size_t)hq, (size_t)d}, dt_of(out_dtype), out);
              auto ws = nn::get_mqa_workspace(*g_ctx, Q, max_len_buf, true);
              nn::multi_query_attention_rag_buffer(*g_ctx, Q, L, KA, VA, M, scale, max_len_buf, O, hq / hkv, -1, ws, SKA, SVA,
                                                   dt_of(out_dtype)))
}

}  // extern "C"
