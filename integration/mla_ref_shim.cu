// TEST INFRASTRUCTURE: extern "C" entry points for the MLA form of nn::multi_query_attention_rag_buffer (dim_head 576,
// one latent head, the same address table as keys and values, a 512-wide output), as the reference's MLA search path
// calls it (src/nn/attention/multi_head_latent_attention.cpp:1053-1068).
//
// integration/Makefile.dropin links this file twice, beside the libraries built from oracle/:
//   * oracle/_ref/libzl_ref_mla.so    against libzl_ref.so    -> the reference's own kernels,
//   * oracle/_ref/libzl_dropin_mla.so against libzl_dropin.so -> integration/zl_nn_dropin.cpp -> libzhilight_b200.so,
// so that tests/mla_golden.py, tests/test_mla_attn_gpu.py and tools/mla_bench.py can run the same reference-signature
// call through both.  The context is the one zlref_init of the linked library created (zlref_ctx).
#include <bmengine/core/core.h>

#include "nn/attention/attention_kernel.h"

#include <cstdio>
#include <vector>

using namespace bmengine;
using core::DataType;
using core::Tensor;

core::Context* zlref_ctx();
char* zlref_err_buf();

namespace {
Tensor wrap(std::vector<size_t> shape, DataType dt, const void* p) {
    size_t n = 1;
    for (auto s : shape) n *= s;
    return Tensor::from_external(shape, dt, const_cast<void*>(p), n * core::get_elem_size(dt), 0, false);
}
DataType dt_of(int code) { return code == 1 ? DataType::kBFloat16 : DataType::kHalf; }

struct MlaCall {
    Tensor Q, L, M, O;
    nn::AttentionWorkspace ws;
    MlaCall(const void* q, const void* buf_lens, const void* mask, size_t mask_len, int max_len_buf, int B, int len_q,
            int hq, int dtype, void* out) {
        const DataType dt = dt_of(dtype);
        Q = wrap({(size_t)B, (size_t)len_q, (size_t)hq, 576}, dt, q);
        L = wrap({(size_t)B}, DataType::kInt32, buf_lens);
        M = wrap({mask_len}, DataType::kInt8, mask);
        O = wrap({(size_t)B, (size_t)len_q, (size_t)hq, 512}, dt, out);
        ws = nn::get_mqa_workspace(*zlref_ctx(), Q, max_len_buf, false);
    }
    void run(const void* kv_table, float scale, int max_len_buf) {
        Tensor KA = wrap({Q.size(0)}, DataType::kDouble, kv_table);
        nn::multi_query_attention_rag_buffer(*zlref_ctx(), Q, L, KA, KA, M, scale, max_len_buf, O, (int)Q.size(2), -1, ws);
    }
};
}  // namespace

#define ZLMLA_TRY(...)                                                                     \
    try {                                                                                  \
        if (!zlref_ctx()) throw std::runtime_error("zlref_init has not run");              \
        __VA_ARGS__;                                                                       \
        BM_CUDART_ASSERT(cudaStreamSynchronize(zlref_ctx()->current_stream()->ptr));       \
        return 0;                                                                          \
    } catch (const std::exception& e) {                                                    \
        snprintf(zlref_err_buf(), 1024, "%s", e.what());                                   \
        return -1;                                                                         \
    }

extern "C" {

// q (B, len_q, hq, 576); kv_table (B) device table of per-task latent caches (len_b, 576); mask the int8 ragged concat of
// (len_q, len_b) (the reference always reads it); out (B, len_q, hq, 512)
int zlref_mqa_rag_buffer_mla(const void* q, const void* buf_lens, const void* kv_table, const void* mask, size_t mask_len,
                             float scale, int max_len_buf, int B, int len_q, int hq, int dtype, void* out) {
    ZLMLA_TRY(MlaCall c(q, buf_lens, mask, mask_len, max_len_buf, B, len_q, hq, dtype, out); c.run(kv_table, scale, max_len_buf))
}

// the same call timed with CUDA events on the context's stream: `iters` launches cycling over n_rot latent-cache tables
// (kv_tables: host array of device tables), after 3 warm-up launches
int zlref_time_mqa_rag_buffer_mla(const void* q, const void* buf_lens, void* const* kv_tables, int n_rot, const void* mask,
                                  size_t mask_len, float scale, int max_len_buf, int B, int len_q, int hq, int dtype, void* out,
                                  int iters, float* us) {
    ZLMLA_TRY(MlaCall c(q, buf_lens, mask, mask_len, max_len_buf, B, len_q, hq, dtype, out);
              auto st = zlref_ctx()->current_stream()->ptr; cudaEvent_t e0, e1;
              BM_CUDART_ASSERT(cudaEventCreate(&e0)); BM_CUDART_ASSERT(cudaEventCreate(&e1));
              for (int i = 0; i < 3; ++i) c.run(kv_tables[i % n_rot], scale, max_len_buf);
              BM_CUDART_ASSERT(cudaEventRecord(e0, st));
              for (int i = 0; i < iters; ++i) c.run(kv_tables[i % n_rot], scale, max_len_buf);
              BM_CUDART_ASSERT(cudaEventRecord(e1, st)); BM_CUDART_ASSERT(cudaEventSynchronize(e1));
              float ms = 0.f; BM_CUDART_ASSERT(cudaEventElapsedTime(&ms, e0, e1)); *us = ms * 1e3f / iters;
              cudaEventDestroy(e0); cudaEventDestroy(e1))
}

}  // extern "C"
