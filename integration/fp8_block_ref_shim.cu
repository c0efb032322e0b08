// TEST INFRASTRUCTURE: an extern "C" entry point for nn::fp8::per_token_cast_to_fp8 (src/nn/quant/fp8/fp8.h:25-30), the
// activation quantisation of Fp8Block::forward (QuantType 10, src/nn/linear/linear.cpp:1697-1960).
//
// integration/Makefile.dropin links this file twice, beside the libraries built from oracle/:
//   * oracle/_ref/libzl_ref_fp8.so    against libzl_ref.so    -> the reference's own KERNEL_per_token_cast_to_fp8,
//   * oracle/_ref/libzl_dropin_fp8.so against libzl_dropin.so -> integration/zl_nn_dropin.cpp -> libzhilight_b200.so,
// so that tests/fp8_block_golden.py and tests/test_fp8_block_gpu.py can run the same reference-signature call through
// both.  The context is the one zlref_init of the linked library created (zlref_ctx).
#include <bmengine/core/core.h>

#include "nn/quant/fp8/fp8.h"

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
}  // namespace

// x (M, K) f16 (dtype 0) or bf16 (1); out_q (M, K) e4m3 bytes; out_scale (K/128, round_up(M, 4)) f32 when col_major,
// (round_up(M, 4), K/128) otherwise -- the scale tensor per_token_cast_to_fp8 attaches to its output, copied out whole.
extern "C" int zlfp8_per_token_cast(const void* x, int M, int K, int dtype, int col_major, void* out_q, void* out_scale) {
    try {
        if (!zlref_ctx()) throw std::runtime_error("zlref_init has not run");
        core::Context& ctx = *zlref_ctx();
        Tensor X = wrap({(size_t)M, (size_t)K}, dtype == 1 ? DataType::kBFloat16 : DataType::kHalf, x);
        Tensor q = nn::fp8::per_token_cast_to_fp8(ctx, X, col_major != 0);
        const cudaStream_t st = ctx.current_stream()->ptr;
        BM_CUDART_ASSERT(cudaMemcpyAsync(out_q, q.data(), (size_t)M * K, cudaMemcpyDeviceToDevice, st));
        const Tensor& s = *q.quant_scale;
        BM_CUDART_ASSERT(cudaMemcpyAsync(out_scale, s.data(), s.nbytes(), cudaMemcpyDeviceToDevice, st));
        BM_CUDART_ASSERT(cudaStreamSynchronize(st));
        return 0;
    } catch (const std::exception& e) {
        snprintf(zlref_err_buf(), 1024, "%s", e.what());
        return -1;
    }
}
