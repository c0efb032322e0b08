// Drop-in definitions of the reference's hot-path operator symbols (namespaces nn, nn::gptq, nn::fp8, int8_op) on top of
// the C-ABI of libzhilight_b200.so -- the file a ZhiLight maintainer adds to the `backend` target in place of the
// corresponding .cu files (INTEGRATION.md).  It is compiled against the reference's own headers where they lie
// in a reference checkout (integration/Makefile.dropin) and linked with bmengine's core + oracle/ref_shim.cu into
// oracle/_ref/libzl_dropin.so, so that tests/test_dropin_gpu.py can drive the reference-signature functions and
// compare them with the reference's own kernels (oracle/_ref/libzl_ref.so) call for call.
//
// Signatures: src/nn/quant/gptq/gptq.h:24-110, src/nn/attention/attention_kernel.h:64-80,
// src/nn/layernorm/layernorm.h:7-34, src/nn/block/block_kernel.h, src/nn/linear/activation_kernel.h:12-16,
// src/nn/position/rotary_embedding.h:52-65, src/kvcache/ragged_buffer_kernel.h:27-36,
// src/nn/quant/int8/quant_kernel.h:15-128, src/nn/quant/fp8/fp8.h:13-30, 3rd/deep_gemm/deep_gemm_api.h.
#include <bmengine/core/core.h>
#include <bmengine/functions/typecast.h>

#include "kvcache/ragged_buffer_kernel.h"
#include "nn/attention/attention_kernel.h"
#include "nn/block/block_kernel.h"
#include "nn/layernorm/layernorm.h"
#include "nn/linear/activation_kernel.h"
#include "nn/position/rotary_embedding.h"
#include "nn/position/rope_preparer.h"
#include "nn/quant/fp8/fp8.h"
#include "nn/quant/gptq/gptq.h"
#include "nn/quant/int8/quant_kernel.h"

#include "zhilight_b200.h"

#include <algorithm>
#include <string>
#include <tuple>

using namespace bmengine;
using core::DataType;
using core::Tensor;

namespace {

// a non-zero C-ABI return code becomes the reference's exception type (exception.h:25-130)
#define ZL_THROW_IF(expr)                                                       \
    do {                                                                        \
        if ((expr) != ZL_OK) BM_EXCEPTION(std::string("zhilight_b200: ") + zl_last_error()); \
    } while (0)

inline int zl_dt(DataType t) {
    if (t == DataType::kHalf) return ZL_F16;
    if (t == DataType::kBFloat16) return ZL_BF16;
    if (t == DataType::kFloat) return ZL_F32;
    BM_EXCEPTION("zhilight_b200: unsupported dtype");
    return -1;
}
inline zl_stream_t st(const core::Context& ctx) { return ctx.current_stream()->ptr; }
inline size_t rows_of(const Tensor& t) { return t.numel() / t.size(-1); }

}  // namespace

// ------------------------------------------------------------------------------------------------------------
// GPTQ / AWQ load-time transforms and the W4A16 GEMMs
// ------------------------------------------------------------------------------------------------------------
namespace nn::gptq {

void gptq_shuffle(const core::Context& ctx, Tensor& q_weight, Tensor q_perm) {
    const int K = (int)q_weight.size(0) * 8, N = (int)q_weight.size(1);
    Tensor scratch = q_perm.numel() ? ctx.tensor(q_weight.shape(), q_weight.dtype()) : Tensor();
    ZL_THROW_IF(zl_gptq_shuffle(q_weight.mutable_data<uint32_t>(), q_perm.numel() ? q_perm.data<int32_t>() : nullptr,
                                scratch.numel() ? scratch.mutable_data<uint32_t>() : nullptr, K, N, st(ctx)));
}

void increase_zero(const core::Context& ctx, Tensor& input) {
    ZL_THROW_IF(zl_gptq_increase_zero(input.mutable_data<uint32_t>(), input.numel(), st(ctx)));
}

void subtract8(const core::Context& ctx, Tensor& input) {
    ZL_THROW_IF(zl_gptq_subtract8(input.mutable_data<uint32_t>(), input.numel(), st(ctx)));
}

void un_shuffle(const core::Context& ctx, Tensor& input) {
    ZL_THROW_IF(zl_awq_un_shuffle(input.mutable_data<uint32_t>(), (int)input.size(0), (int)input.size(1), st(ctx)));
}

Tensor shuffle_awq(const core::Context& ctx, Tensor& input, bool use_exllama) {
    const int K = (int)input.size(0), N = (int)input.size(1) * 8;
    Tensor out = ctx.tensor({(size_t)K / 8, (size_t)N}, DataType::kInt32);
    ZL_THROW_IF(zl_awq_shuffle(input.data<uint32_t>(), out.mutable_data<uint32_t>(), K, N, use_exllama ? 1 : 0, st(ctx)));
    return out;
}

Tensor q4_to_q8(const core::Context& ctx, const Tensor& input) {
    auto shape = input.shape();
    shape[shape.size() - 1] *= 8;
    Tensor out = ctx.tensor(shape, DataType::kInt8);
    ZL_THROW_IF(zl_q4_to_q8(input.data<uint32_t>(), out.mutable_data<uint8_t>(), input.numel(), st(ctx)));
    return out;
}

Tensor dequant_k_major(const core::Context& ctx, const Tensor& q_weight, const Tensor& qzeros, const Tensor& scales,
                       int out_type) {
    BM_ASSERT_EQ(out_type, 0, "only the fp16 form is provided");
    const int N = (int)q_weight.size(0), K = (int)q_weight.size(1) * 8, G = (int)scales.size(1);
    Tensor out = ctx.tensor({(size_t)N, (size_t)K}, DataType::kHalf);
    ZL_THROW_IF(zl_gptq_dequant_k_major(q_weight.data<uint32_t>(), qzeros.data<uint8_t>(), scales.data(), out.data(), N, K,
                                        K / G, st(ctx)));
    return out;
}

namespace {
// In the real integration the ZLW4I blob is built once in Int4GPTQ::preprocess_weight and rides on
// q_weight.quant_scale (tensor.h:32-35).  This stand-alone wrapper packs per call when that twin is absent.
Tensor packed_of(const core::Context& ctx, const Tensor& q_weight, const Tensor& qzeros, const Tensor& scales, bool sym,
                 const int32_t* row_map, int n_rows, int variant) {
    if (q_weight.quant_scale && row_map == nullptr) return *q_weight.quant_scale;
    const int K = (int)q_weight.size(-1) * 8, G = (int)scales.size(-1);
    const size_t bytes = zl_w4_packed_bytes(n_rows, K, K / G);
    BM_ASSERT(bytes > 0, "shape not supported by the ZLW4 layout (N % 32, K % 128, group 128)");
    Tensor packed = ctx.tensor({bytes}, DataType::kInt8);
    ZL_THROW_IF(zl_w4_pack_v(q_weight.data<uint32_t>(), qzeros.data<uint8_t>(), scales.data(), row_map, packed.data(),
                             n_rows, K, K / G, sym ? 1 : 0, variant, st(ctx)));
    return packed;
}
}  // namespace

Tensor gptq_gemm_k_major(const core::Context& ctx, const Tensor& a, const Tensor& q_weight, const Tensor& qzeros,
                         const Tensor& scales, const Tensor& q_perm, const Tensor& rev_perm, const Tensor* bias, bool sym,
                         bool cache_only, Tensor* output, const Tensor* precomputed_w8) {
    (void)rev_perm;
    (void)precomputed_w8;
    BM_ASSERT_EQ(a.dtype(), DataType::kHalf, "A must be half");             // q_gemm_k_major.cu:989
    BM_ASSERT(qzeros.dtype() == DataType::kInt8, "qzeros must be int8");     // :990
    BM_ASSERT_EQ(q_perm.numel(), 0, "act-order is not supported on the H100 path");
    const int K = (int)a.size(-1), M = (int)(a.numel() / K), N = (int)q_weight.size(-2);
    BM_ASSERT_EQ((size_t)K, q_weight.size(-1) * 8, "K mismatch");
    if (cache_only) return Tensor();
    auto shape = a.shape();
    shape[shape.size() - 1] = N;
    Tensor c = output ? *output : ctx.tensor(shape, a.dtype());
    const int variant = zl_w4_int_kernel_fits(M < 32 ? M : 32, N, K) ? 1 : 0;
    Tensor packed = packed_of(ctx, q_weight, qzeros, scales, sym, nullptr, N, variant);
    zl_w4_fused_args_t args = {};
    args.x = a.data();
    args.ldx = K;
    args.packed = packed.data();
    args.bias = bias && bias->numel() ? bias->data() : nullptr;
    args.y = c.data();
    args.M = M;
    args.N = N;
    args.K = K;
    args.group_size = K / (int)scales.size(-1);
    args.epilogue = ZL_EPI_NONE;
    args.variant = variant;
    ZL_THROW_IF(zl_w4a16_gemm_fused(&args, st(ctx)));
    return c;
}

Tensor gemm_fuse_gate_in(const core::Context& ctx, const Tensor& a, const Tensor& q_weight1, const Tensor& qzeros1,
                         const Tensor& scales1, const Tensor& rev_perm1, const Tensor& q_weight2, const Tensor& qzeros2,
                         const Tensor& scales2, const Tensor& rev_perm2, bool sym) {
    (void)rev_perm1;
    (void)rev_perm2;
    BM_ASSERT_EQ(a.dtype(), DataType::kHalf, "A must be half");
    const int K = (int)a.size(-1), M = (int)(a.numel() / K), F = (int)q_weight1.size(-2), G = (int)scales1.size(-1);
    // gate rows then up rows in one k-major tensor; the row map interleaves them per MMA tile (SwiGLU epilogue)
    auto cat = [&](const Tensor& x, const Tensor& y, DataType dt, size_t cols) {
        Tensor o = ctx.tensor({(size_t)2 * F, cols}, dt);
        BM_CUDART_ASSERT(cudaMemcpyAsync(o.data(), x.data(), x.nbytes(), cudaMemcpyDeviceToDevice, st(ctx)));
        BM_CUDART_ASSERT(cudaMemcpyAsync(o.data<char>() + x.nbytes(), y.data(), y.nbytes(), cudaMemcpyDeviceToDevice, st(ctx)));
        return o;
    };
    Tensor qw = cat(q_weight1, q_weight2, DataType::kInt32, (size_t)K / 8);
    Tensor qz = cat(qzeros1, qzeros2, DataType::kInt8, (size_t)G);
    Tensor sc = cat(scales1, scales2, DataType::kHalf, (size_t)G);
    // packed row p <- source row (zhilight_b200/ops.py::swiglu_row_map): 16-row groups of 8 gate rows then 8 up rows
    std::vector<int32_t> map(2 * (size_t)F);
    for (int p = 0; p < 2 * F; ++p) {
        const int t16 = p / 16, r = p % 16;
        map[p] = r < 8 ? t16 * 8 + r : F + t16 * 8 + (r - 8);
    }
    Tensor d_map = ctx.tensor({map.size()}, DataType::kInt32);
    d_map.from_buffer(map.data());
    const int variant = zl_w4_int_kernel_fits(M < 32 ? M : 32, 2 * F, K) ? 1 : 0;
    Tensor packed = packed_of(ctx, qw, qz, sc, sym, d_map.data<int32_t>(), 2 * F, variant);
    auto shape = a.shape();
    shape[shape.size() - 1] = F;
    Tensor c = ctx.tensor(shape, a.dtype());
    zl_w4_fused_args_t args = {};
    args.x = a.data();
    args.ldx = K;
    args.packed = packed.data();
    args.y = c.data();
    args.M = M;
    args.N = 2 * F;
    args.K = K;
    args.group_size = K / G;
    args.epilogue = ZL_EPI_SWIGLU;
    args.variant = variant;
    ZL_THROW_IF(zl_w4a16_gemm_fused(&args, st(ctx)));
    return c;
}

}  // namespace nn::gptq

// ------------------------------------------------------------------------------------------------------------
// norm / residual / activation / RoPE / KV append / decode attention
// ------------------------------------------------------------------------------------------------------------
namespace nn {

class LayerNorm::impl {
public:
    Tensor weight;
    float eps, scale;
    impl(const core::Context& ctx, unsigned dim_model, float eps_, float scale_, DataType dtype)
        : weight(ctx.parameter({dim_model}, dtype)), eps(eps_), scale(scale_) {}
};

LayerNorm::LayerNorm(const core::Context& ctx, int dim_model, bool quant, float eps, float scale, DataType dtype,
                     int num_head)
    : core::Layer() {
    BM_ASSERT(!quant && num_head == 1, "drop-in LayerNorm covers the plain RMSNorm of the decode path");
    pimpl.reset(new impl(ctx, (unsigned)dim_model, eps, scale, dtype));
    add_parameter("weight", pimpl->weight);
}
LayerNorm::~LayerNorm() = default;

Tensor LayerNorm::forward(const core::Context& ctx, const Tensor& x) {
    Tensor y = ctx.tensor(x.shape(), x.dtype());
    ZL_THROW_IF(zl_rmsnorm(x.data(), pimpl->weight.data(), y.data(), (int)rows_of(x), (int)x.size(-1), pimpl->eps,
                           pimpl->scale, zl_dt(x.dtype()), 0, st(ctx)));
    return y;
}

Tensor LayerNorm::fuse_add(const core::Context& ctx, const Tensor& a, const Tensor& b, Tensor& c) {
    Tensor y = ctx.tensor(a.shape(), a.dtype());
    ZL_THROW_IF(zl_add_rmsnorm(a.data(), b.data(), pimpl->weight.data(), c.data(), y.data(), (int)rows_of(a),
                               (int)a.size(-1), pimpl->eps, pimpl->scale, /*mode=*/1, zl_dt(a.dtype()), 0, st(ctx)));
    return y;
}

void LayerNorm::inplace(const core::Context& ctx, Tensor& x) {
    ZL_THROW_IF(zl_rmsnorm(x.data(), pimpl->weight.data(), x.data(), (int)rows_of(x), (int)x.size(-1), pimpl->eps,
                           pimpl->scale, zl_dt(x.dtype()), 0, st(ctx)));
}

void LayerNorm::forward_2(const core::Context& ctx, Tensor& x, Tensor& y, Tensor& x_out, Tensor& y_out, LayerNorm* la,
                          LayerNorm* lb) {
    x_out = la->forward(ctx, x);
    y_out = lb->forward(ctx, y);
}

void LayerNorm::set_rms(bool b) { BM_ASSERT(b, "only RMSNorm is on the decode path"); }

void LayerNorm::load_state_dict(const core::Context& ctx, const std::map<std::string, const Tensor>& state_dict,
                                const std::string& prefix, bool allow_missing) {
    (void)allow_missing;
    ctx.load_parameter(&pimpl->weight, prefix + ".weight", state_dict, false, core::DistLayout::REPLICATED);
}

void element_add_scale_out(const core::Context& ctx, const Tensor& a, const Tensor& b, Tensor& c, float scale,
                           bool scale_residual) {
    BM_ASSERT(!scale_residual || scale == 1.f, "decode path uses scale_residual = false (block.cpp:125,140)");
    ZL_THROW_IF(zl_element_add_scale(a.data(), b.data(), c.data(), a.numel(), scale, zl_dt(a.dtype()), st(ctx)));
}

Tensor element_add_scale(const core::Context& ctx, const Tensor& a, const Tensor& b, float scale, bool scale_residual) {
    Tensor c = ctx.tensor(a.shape(), a.dtype());
    element_add_scale_out(ctx, a, b, c, scale, scale_residual);
    return c;
}

void gate_mul_inplace(const core::Context& ctx, Tensor& inp, const Tensor& in2, const std::string& gate_type) {
    const int act = gate_type == "gelu" ? 1 : 0;
    const int F = (int)inp.size(-1), T = (int)rows_of(inp);
    ZL_THROW_IF(zl_gate_mul(inp.data(), F, in2.data(), F, inp.data(), F, T, F, act, zl_dt(inp.dtype()), st(ctx)));
}

void rope_qk_cache(const core::Context& ctx, const Tensor& cos, const Tensor& sin, const Tensor& in, Tensor& out_q,
                   Tensor& out_k, Tensor& out_v, size_t num_heads, size_t num_kv_heads, size_t dim_head, DataType dtype,
                   bool neox_style) {
    const size_t T = in.size(0);
    out_q = ctx.tensor({T, num_heads * dim_head}, dtype);
    out_k = ctx.tensor({T, num_kv_heads * dim_head}, dtype);
    out_v = ctx.tensor({T, num_kv_heads * dim_head}, dtype);
    ZL_THROW_IF(zl_rope_qk_cache(cos.data<float>(), sin.data<float>(), in.data(), out_q.data(), out_k.data(), out_v.data(),
                                 (int)T, (int)num_heads, (int)num_kv_heads, (int)dim_head, neox_style ? 1 : 0, zl_dt(dtype),
                                 st(ctx)));
}

void copy_to_rag_buffer2(const core::Context& ctx, const Tensor& placement, const Tensor& buf_lens, const Tensor& k_src,
                         const Tensor& v_src, Tensor* buf_k_addr, Tensor* buf_v_addr, bool is_scale) {
    BM_ASSERT(!is_scale, "int8 KV scales are not on this path");
    const int B = (int)k_src.size(0), len_q = (int)k_src.size(1), hkv = (int)k_src.size(2), d = (int)k_src.size(3);
    ZL_THROW_IF(zl_copy_to_rag_buffer2(placement.data<int32_t>(), buf_lens.data<int32_t>(), k_src.data(), v_src.data(),
                                       buf_k_addr->data<void*>(), buf_v_addr->data<void*>(), B, len_q, hkv, d,
                                       ctx.is_BSHD() ? 1 : 0, zl_dt(k_src.dtype()), st(ctx)));
}

void multi_query_attention_rag_buffer(const core::Context& ctx, const Tensor& batch_q, const Tensor& buf_lens,
                                      const Tensor& key_buf_addrs, const Tensor& val_buf_addrs, const Tensor& mask,
                                      const float scale, const int max_len_buf, Tensor& output, const int m_query,
                                      int algo_id, const AttentionWorkspace& ws, const Tensor& scale_key_addrs,
                                      const Tensor& scale_val_addrs, DataType dequant_dtype) {
    (void)algo_id;
    (void)ws;
    const int B = (int)batch_q.size(0), len_q = (int)batch_q.size(1), Hq = (int)batch_q.size(2), d = (int)batch_q.size(3);
    if (d == 576) {
        // MLA (multi_head_latent_attention.cpp:1053-1068): one latent head whose 576-wide rows are K and whose first 512
        // elements are V; the reference passes the same address table as keys and values
        BM_ASSERT_EQ(output.size(-1), 512, "dim_head mismatch");
        BM_ASSERT_EQ(m_query, Hq, "MLA attends one latent head");
        BM_ASSERT(key_buf_addrs.data() == val_buf_addrs.data(), "MLA keys and values share one latent cache");
        BM_ASSERT(!scale_key_addrs.numel(), "no int8 latent cache");
        const size_t mwsb = zl_mla_decode_attention_workspace_bytes(B, len_q, Hq, max_len_buf);
        Tensor mwork = ctx.tensor({std::max<size_t>(mwsb, 16)}, DataType::kInt8);
        ZL_THROW_IF(zl_mla_decode_attention(batch_q.data(), buf_lens.data<int32_t>(), key_buf_addrs.data<void*>(),
                                            mask.numel() ? mask.data<int8_t>() : nullptr, scale, max_len_buf,
                                            output.data(), B, len_q, Hq, mwork.data(), mwsb, zl_dt(batch_q.dtype()), 0,
                                            st(ctx)));
        return;
    }
    const size_t wsb = zl_decode_attention_workspace_bytes(B, len_q, Hq, d, max_len_buf);
    Tensor work = ctx.tensor({wsb}, DataType::kInt8);
    if (scale_key_addrs.numel()) {
        // int8 KV cache (KERNEL_mqa_rag_buffer_split_kv_quant, attention_kernel.cu:804-880): uint8 codes + fp32 scales
        BM_ASSERT_EQ(batch_q.dtype(), DataType::kHalf, "input must be half");
        BM_ASSERT(ctx.is_BSHD(), "int8 KV cache is BSHD");
        ZL_THROW_IF(zl_decode_attention_kv8(batch_q.data(), buf_lens.data<int32_t>(), key_buf_addrs.data<void*>(),
                                            val_buf_addrs.data<void*>(), scale_key_addrs.data<void*>(),
                                            scale_val_addrs.data<void*>(), mask.numel() ? mask.data<int8_t>() : nullptr, scale,
                                            max_len_buf, output.data(), B, len_q, Hq, Hq / m_query, d, work.data(), wsb,
                                            zl_dt(dequant_dtype), 0, st(ctx)));
        return;
    }
    ZL_THROW_IF(zl_decode_attention(batch_q.data(), buf_lens.data<int32_t>(), key_buf_addrs.data<void*>(),
                                    val_buf_addrs.data<void*>(), mask.numel() ? mask.data<int8_t>() : nullptr, scale,
                                    max_len_buf, output.data(), B, len_q, Hq, Hq / m_query, d, ctx.is_BSHD() ? 1 : 0,
                                    work.data(), wsb, zl_dt(batch_q.dtype()), 0, st(ctx)));
}

// the reference sizes its split workspace here (attention_kernel.cu:1237-1250); ours is allocated inside the wrapper above
AttentionWorkspace get_mqa_workspace(const core::Context& ctx, const Tensor& batch_q, int max_len_buf, bool is_quantized) {
    (void)max_len_buf;
    (void)is_quantized;
    const size_t vheads = batch_q.numel() / batch_q.size(-1);
    return {ctx.tensor({vheads, 1, batch_q.size(-1)}, DataType::kFloat), ctx.tensor({vheads, 1}, DataType::kFloat),
            ctx.tensor({vheads, 1}, DataType::kFloat)};
}

// RopePreparer (rope_preparer.cu:49-233): cos / sin tables, plain and llama3 wavelength scaling
class RopePreparer::impl {
public:
    model::ModelConfig cfg;
    explicit impl(model::ModelConfig c) : cfg(std::move(c)) {}
};
RopePreparer::RopePreparer(const core::Context& ctx, model::ModelConfig cfg) : pimpl(new impl(std::move(cfg))) { (void)ctx; }
RopePreparer::~RopePreparer() {}
std::tuple<Tensor, Tensor> RopePreparer::forward(const core::Context& ctx, const Tensor& tokens, const Tensor& pos) {
    (void)tokens;
    const model::ModelConfig& c = pimpl->cfg;
    const int d = c.qk_rope_head_dim > 0 ? c.qk_rope_head_dim : c.dim_head;
    auto shape = pos.shape();
    shape.push_back((size_t)d);
    Tensor cos = ctx.tensor(shape, DataType::kFloat), sin = ctx.tensor(shape, DataType::kFloat);
    const bool l3 = c.rope_cfg.type == "llama3";
    if (!l3 && c.rope_cfg.type != "") throw std::runtime_error("RopePreparer: Not implemented rope type: " + c.rope_cfg.type);
    ZL_THROW_IF(zl_rope_cos_sin(pos.data<int32_t>(), cos.mutable_data<float>(), sin.mutable_data<float>(), (int)pos.numel(), d,
                                c.rope_theta, l3 ? c.rope_cfg.factor : 0.f, c.rope_cfg.low_freq_factor,
                                c.rope_cfg.high_freq_factor, (float)c.rope_cfg.original_max_position,
                                c.rope_cfg.neox_style ? 1 : 0, st(ctx)));
    return {cos, sin};
}

}  // namespace nn

// ------------------------------------------------------------------------------------------------------------
// INT8 / FP8 activation quantisation, scale-back, int8 TP-reduce stages
// ------------------------------------------------------------------------------------------------------------
namespace int8_op {

void quant_calc_scale(const core::Context& ctx, const Tensor& input, Tensor* output, Tensor* output_scale, int q_max,
                      int q_zero) {
    BM_ASSERT(q_max == 127 && (q_zero == 0 || q_zero == 128), "per-token int8 (q_zero 0) or the uint8 KV-cache form (q_zero 128)");
    const int K = (int)input.size(-1), M = (int)rows_of(input);
    if (output->shape() != input.shape()) *output = ctx.tensor(input.size(), DataType::kInt8);
    if (output_scale->numel() != (size_t)M) *output_scale = ctx.tensor({(size_t)M}, DataType::kFloat);
    if (q_zero == 128) {
        ZL_THROW_IF(zl_int8_quant_rows_u8(input.data(), output->data(), output_scale->mutable_data<float>(), M, K,
                                          zl_dt(input.dtype()), st(ctx)));
        return;
    }
    ZL_THROW_IF(zl_int8_quant_per_token(input.data(), K, output->data(), output_scale->mutable_data<float>(), M, K,
                                        zl_dt(input.dtype()), 0, st(ctx)));
}

Tensor quant_calc_scale(const core::Context& ctx, const Tensor& input, int q_max, int q_zero) {
    Tensor q, s;
    quant_calc_scale(ctx, input, &q, &s, q_max, q_zero);
    set_quant_scale(q, s);
    return q;
}

void set_quant_scale(Tensor& tensor, const Tensor& quant_scale) {
    tensor.quant_scale = std::make_shared<Tensor>();
    *tensor.quant_scale = quant_scale;
}

void layernorm_quant(const core::Context& ctx, const Tensor& input, const Tensor& weight, Tensor* output,
                     Tensor* output_int8, Tensor* output_scale, float eps, float scale) {
    const int D = (int)input.size(-1), T = (int)rows_of(input);
    if (output->shape() != input.shape()) *output = ctx.tensor(input.size(), input.dtype());
    if (output_int8->shape() != input.shape()) *output_int8 = ctx.tensor(input.size(), DataType::kInt8);
    if (output_scale->numel() != (size_t)T) *output_scale = ctx.tensor({(size_t)T}, DataType::kFloat);
    BM_ASSERT_EQ(output_scale->dtype(), DataType::kFloat, "float scales");
    ZL_THROW_IF(zl_rmsnorm_quant(input.data(), weight.data(), output->data(), output_int8->data(),
                                 output_scale->mutable_data<float>(), T, D, eps, scale, zl_dt(input.dtype()), 0, st(ctx)));
}

std::tuple<Tensor, Tensor> quant_group_32(const core::Context& ctx, const Tensor& input) {
    const size_t M = input.numel() / 32;
    Tensor q = ctx.tensor(input.shape(), DataType::kInt8);
    Tensor s = ctx.tensor({M}, input.dtype());
    ZL_THROW_IF(zl_quant_group_32(input.data(), q.mutable_data<int8_t>(), s.data(), M, zl_dt(input.dtype()), st(ctx)));
    return {q, s};
}

void dequant_sum_quant_g32(const core::Context& ctx, const Tensor& my, const Tensor& q_others, const Tensor& scale_others,
                           Tensor* q_sum, Tensor* scale_sum) {
    const size_t M = my.numel() / 32;
    const int ws = (int)q_others.size(0) + 1;
    ZL_THROW_IF(zl_dequant_sum_quant_g32(my.data(), q_others.data<int8_t>(), scale_others.data(),
                                         q_sum->mutable_data<int8_t>(), scale_sum->data(), M, ws, zl_dt(my.dtype()), st(ctx)));
}

void dequant_group_32(const core::Context& ctx, const Tensor& q, const Tensor& scale, Tensor* out) {
    ZL_THROW_IF(zl_dequant_group_32(q.data<int8_t>(), scale.data(), nullptr, out->data(), q.numel() / 32,
                                    zl_dt(scale.dtype()), st(ctx)));
}

Tensor dequant_group_fuse_add(const core::Context& ctx, const Tensor& q, const Tensor& scale, const Tensor& c) {
    Tensor out = ctx.tensor(c.shape(), c.dtype());
    ZL_THROW_IF(zl_dequant_group_32(q.data<int8_t>(), scale.data(), c.data(), out.data(), q.numel() / 32,
                                    zl_dt(scale.dtype()), st(ctx)));
    return out;
}

// Int8Linear's stock forward still holds an int32 accumulator here (linear.cpp:627); the fused zl_w8a8_gemm makes this
// call disappear once Int8Linear::forward is switched over (INTEGRATION.md 1b).
Tensor quant_scale_back(const core::Context& ctx, const Tensor& input, const Tensor* scale_x, const Tensor* scale_y,
                        DataType out_type, Tensor* output) {
    BM_ASSERT_EQ(input.dtype(), DataType::kInt32, "Wrong input dtype");
    if (scale_y->dtype() != DataType::kFloat) out_type = scale_y->dtype();
    const int N = (int)input.size(-1), M = (int)rows_of(input);
    Tensor ret = output ? *output : ctx.tensor(input.size(), out_type);
    ZL_THROW_IF(zl_int8_scale_back(input.data<int32_t>(), scale_x->data<float>(), scale_y->data(), zl_dt(scale_y->dtype()),
                                   ret.data(), M, N, zl_dt(out_type), st(ctx)));
    return ret;
}

}  // namespace int8_op

namespace nn::fp8 {

Tensor dynamic_scaled_quant(const core::Context& ctx, const Tensor& input, float MAX_E4M3) {
    BM_ASSERT(MAX_E4M3 == 448.f, "e4m3 max");
    Tensor out = ctx.tensor(input.shape(), DataType::kInt8, "", std::max<size_t>(32 * input.size(-1), 1024));
    Tensor scale = ctx.tensor({1}, DataType::kFloat);
    ZL_THROW_IF(zl_fp8_quant_per_tensor(input.data(), out.data(), scale.mutable_data<float>(), input.numel(),
                                        zl_dt(input.dtype()), 0, st(ctx)));
    out.quant_scale = std::make_shared<Tensor>();
    *out.quant_scale = scale;
    return out;
}

// fp8_util.cu:231-322: one scale per (token, 128 columns), (K/128, round_up(M, 4)) column-major or (round_up(M, 4),
// K/128) row-major.  The kernel writes column-major; the row-major form is its transpose.
Tensor per_token_cast_to_fp8(const core::Context& ctx, const Tensor& input, bool scale_col_major, float MAX_E4M3) {
    BM_ASSERT(MAX_E4M3 == 448.f, "e4m3 max");
    BM_ASSERT_EQ(input.ndim(), 2, "FP8 block_scale: input is not 2D");
    BM_ASSERT_EQ(input.size(1) % 128, 0, "FP8 block_scale: input.size(1) can't divide 128");
    const size_t m = input.size(0), n = input.size(1), aligned_m = (m + 3) / 4 * 4;
    Tensor out = ctx.tensor(input.shape(), DataType::kFP8_E4M3, "", std::max<size_t>(32 * n, 1024));
    Tensor col = ctx.tensor({n / 128, aligned_m}, DataType::kFloat);
    ZL_THROW_IF(zl_fp8_quant_per_token_group(input.data(), (int)input.stride(0), out.data(), col.mutable_data<float>(),
                                             (int)aligned_m, (int)m, (int)n, zl_dt(input.dtype()), 0, st(ctx)));
    Tensor scale = col;
    if (!scale_col_major) {
        scale = ctx.tensor({aligned_m, n / 128}, DataType::kFloat);
        ZL_THROW_IF(zl_transpose_2d(col.data(), scale.mutable_data(), (int)(n / 128), (int)aligned_m, 4, st(ctx)));
    }
    out.set_quant_scale(scale);
    return out;
}

}  // namespace nn::fp8

// DeepGEMM's entry point (3rd/deep_gemm/deep_gemm_api.h), called by Fp8Block::forward (linear.cpp:1880-1945) with
// lhs = per_token_cast_to_fp8's codes and column-major scales (leading dimension round_up(m, 4)), rhs = the (n, k) e4m3
// weight with (ceil(n/128), k/128) f32 weight_scale_inv, bf16 out.  Plain GEMMs (num_groups == 1) run on
// zl_fp8_block_gemm; the grouped (MoE) form returns -1, which the caller reports as an unsupported shape.
extern "C" int deep_gemm_fp8_block_h20_group(void* lhs, void* lhs_scales, void* rhs, void* rhs_scales, void* out,
                                             void* grouped_layout, void* stream, int m, int n, int k, int block_m,
                                             int num_groups) {
    (void)block_m;
    if (num_groups != 1 || grouped_layout != nullptr) return -1;
    const int rc = zl_fp8_block_gemm(lhs, static_cast<const float*>(lhs_scales), (m + 3) / 4 * 4, rhs,
                                     static_cast<const float*>(rhs_scales), out, m, n, k, ZL_BF16, 0,
                                     static_cast<zl_stream_t>(stream));
    return rc == ZL_OK ? 0 : -1;
}
