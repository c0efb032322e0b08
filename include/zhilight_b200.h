/*
 * zhilight_b200 -- C-ABI of the H100-native (sm_90a) quantized-decode hot path of ZhiLight.
 *
 * Every entry point replaces one reference operator (cited as file:line inside the reference checkout).
 * Conventions (SURVEY.md section 8b):
 *   - plain pointers + sizes, no C++/torch types; all data pointers are DEVICE pointers unless
 *     the name ends in _host;
 *   - stream-ordered on `stream`, no allocation, no host sync inside (except zl_llama_* which
 *     owns its buffers);
 *   - returns ZL_OK (0) or a negative error code; zl_last_error() gives the message of the last
 *     failure on the calling thread.  The C++ mirror (zhilight_b200/host) turns codes into the
 *     reference's BMEngineException behaviour;
 *   - re-entrant per device; no global mutable state besides per-device symmetric buffers
 *     created by zl_comm_*.
 *
 * dtype codes follow bmengine core::DataType ordering where they overlap
 * (3rd/bmengine/bmengine/include/bmengine/core/dtype.h).
 */
#ifndef ZHILIGHT_B200_H_
#define ZHILIGHT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* zl_stream_t; /* == cudaStream_t */

enum {
    ZL_OK = 0,
    ZL_ERR_INVALID_ARG = -1,
    ZL_ERR_UNSUPPORTED = -2,
    ZL_ERR_CUDA = -3,
    ZL_ERR_STATE = -4,
    /* the KV arena (zl_llama_config_t.kv_rows > 0) cannot give a call the rows it writes, even after compaction: nothing
     * was enqueued and the model keeps running, so the caller can release a task (zl_llama_kv_release) and retry */
    ZL_ERR_KV_FULL = -5
};

enum { ZL_F16 = 0, ZL_BF16 = 1, ZL_F32 = 2 };

/* epilogues of zl_w4a16_gemm */
enum {
    ZL_EPI_NONE = 0,     /* y = acc (+bias)                                                     */
    ZL_EPI_SWIGLU = 1,   /* packed rows interleave gate/up; y[:, n] = silu(T(gate)) * T(up)      */
    ZL_EPI_RESIDUAL = 2, /* y = T(T(acc (+bias)) + residual)   (block_kernel.cu:7-17)           */
    ZL_EPI_QKV_ROPE = 3  /* fused qkv: split + RoPE(q,k) + KV append (zl_w4a16_gemm_fused only)    */
};

const char* zl_last_error(void);
int zl_version(void);
/* number of kernel launches issued by this library on the calling thread since the last reset */
long long zl_launch_count(int reset);
/* one-time per-device kernel attribute setup (opt-in shared memory); called by zl_llama_create and lazily
 * by the ops; must not first happen inside a stream capture. */
int zl_prepare(void);

/* ------------------------------------------------------------------------------------------ *
 * Load-time integer layout transforms (bit-exact with the reference)
 * ------------------------------------------------------------------------------------------ */
/* nn::gptq::gptq_shuffle  (src/nn/quant/gptq/q_gemm.cu:778-872, qdq_4.cuh:16-35).
 * qweight (K/8, N) int32 in place.  q_perm (K) int32 or NULL; scratch (K/8*N words) required iff q_perm. */
int zl_gptq_shuffle(uint32_t* qweight, const int32_t* q_perm, uint32_t* scratch, int K, int N,
                    zl_stream_t stream);
/* nn::gptq::increase_zero (src/nn/quant/gptq/utils.cu:61-88): each nibble (z+1)&15, in place. */
int zl_gptq_increase_zero(uint32_t* qzeros, size_t n_words, zl_stream_t stream);
/* nn::gptq::subtract8 (utils.cu:91-118). */
int zl_gptq_subtract8(uint32_t* words, size_t n_words, zl_stream_t stream);
/* nn::gptq::q4_to_q8 (utils.cu:177-214): (R, C/8) int32 -> (R, C) uint8. */
int zl_q4_to_q8(const uint32_t* in, uint8_t* out, size_t n_words, zl_stream_t stream);
/* nn::gptq::un_shuffle (utils.cu:25-58): AWQ zero de-interleave in place, (rows, cols) words. */
int zl_awq_un_shuffle(uint32_t* qzeros, int rows, int cols, zl_stream_t stream);
/* nn::gptq::shuffle_awq (utils.cu:121-174): (K, N/8) -> (K/8, N). */
int zl_awq_shuffle(const uint32_t* in, uint32_t* out, int K, int N, int use_exllama, zl_stream_t stream);
/* functions::Transpose for 2-D tensors of 1/2/4-byte elements: (rows, cols) -> (cols, rows). */
int zl_transpose_2d(const void* in, void* out, int rows, int cols, int elem_bytes, zl_stream_t stream);
/* nn::gptq::dequant_k_major out_type 0 (q_gemm_k_major.cu:843-905): W16[n,k] = half(q-z)*half(s). */
int zl_gptq_dequant_k_major(const uint32_t* qweight_km, const uint8_t* qzeros_km, const void* scales_km,
                            void* out_f16, int N, int K, int group_size, zl_stream_t stream);

/* ------------------------------------------------------------------------------------------ *
 * ZLW4: the tile-packed W4 layout consumed by zl_w4a16_gemm (DESIGN.md section 3).
 * Built once at load from the reference k-major tensors
 * (Int4GPTQ::preprocess_weight, src/nn/linear/linear.cpp:1139-1160).
 * ------------------------------------------------------------------------------------------ */
size_t zl_w4_packed_bytes(int N, int K, int group_size);
/* qweight_km (N_src, K/8) u32 shuffled, qzeros_km (N_src, K/g) u8 (NULL or sym!=0 -> zero 8),
 * scales_km (N_src, K/g) f16.  row_map (N) int32 or NULL: packed row p takes source row row_map[p]. */
int zl_w4_pack(const uint32_t* qweight_km, const uint8_t* qzeros_km, const void* scales_km,
               const int32_t* row_map, void* packed, int N, int K, int group_size, int sym,
               zl_stream_t stream);
/* variant 0: ZLW4 (fp16 HMMA kernels); variant 1: ZLW4I (exact-integer IMMA kernel, zl_w4a16_gemm_fused with
 * args.variant = 1).  zl_w4_pack == variant 0. */
int zl_w4_pack_v(const uint32_t* qweight_km, const uint8_t* qzeros_km, const void* scales_km,
                 const int32_t* row_map, void* packed, int N, int K, int group_size, int sym, int variant,
                 zl_stream_t stream);
int zl_w4_unpack_v(const void* packed, uint32_t* qweight_km, uint8_t* qzeros_km, void* scales_km, int N, int K,
                   int group_size, int variant, zl_stream_t stream);
/* inverse (tests): recover k-major nibbles/zeros/scales from the packed form. */
int zl_w4_unpack(const void* packed, uint32_t* qweight_km, uint8_t* qzeros_km, void* scales_km, int N, int K,
                 int group_size, zl_stream_t stream);

/* nn::gptq::gptq_gemm_k_major / KERNEL_gemm_warp_reduce / gemm_fuse_gate_in
 * (src/nn/quant/gptq/q_gemm_k_major.cu:957-1116, 176-237, 529-578):
 * y[m,n] = sum_k x[m,k] * (q[n,k]-z[n,k/g]) * s[n,k/g] (+bias[n]), fp16 in/out, fp32 accumulate.
 * x (M, K) f16 row stride ldx; y (M, N_out) f16 where N_out = N (NONE/RESIDUAL) or N/2 (SWIGLU).
 * Any M >= 1 (weights are re-streamed per 32-token chunk).  pdl != 0 -> programmatic dependent launch. */
int zl_w4a16_gemm(const void* x, int ldx, const void* packed, const void* bias, const void* residual,
                  void* y, int M, int N, int K, int group_size, int epilogue, int pdl, zl_stream_t stream);

/* The same GEMM with the neighbouring operators of the decode layer folded in (DESIGN.md section 4.1):
 *   ln_weight != NULL : nn::LayerNorm (rms, layernorm.cu:9-42) of x is fused into the prologue:
 *                       y = rsqrt(mean(x^2)+eps) * (W . (x*ln_weight)) (+bias);
 *   epilogue ZL_EPI_QKV_ROPE: W is the fused qkv weight packed with zl_qkv_rope_row_map; the epilogue applies
 *                       rope_qk_cache (rotary_embedding_fuse_cache.cu:23-63) and copy_to_rag_buffer2
 *                       (ragged_buffer_kernel.cu:194-222, BSHD) and writes q (M, num_heads*dim_head).
 *   tp_mode (tensor parallel, integer kernel only; replaces ModelContext::reduce_sum + element_add_scale between a
 *                       row-parallel Linear and the next column-parallel one, model_context.cpp:203-243, block.cpp:123-141):
 *                       2 on the row-parallel GEMM (o_proj / w_out, epilogue NONE, y unused): the fp16 partial tile is
 *                       stored straight into every rank's NVLink-mapped inbox of tp_comm as 8-byte words {2 x fp16, tag}
 *                       (valid on arrival: no flags, no fences);
 *                       1 on the next GEMM: its activation row becomes T(T(sum_r partial_r) + x), x = residual stream,
 *                       reduced in rank order while the activations are staged (the staging loop polls the words' tags);
 *                       the sum is also stored to tp_h_out (M, K; must not alias x).  0: off.
 *                       tp_index: index of the exchange within the step (0 .. 511, consecutive, the same on producer and
 *                       consumer), | 512 when the step has an ODD number of exchanges (the two slots must alternate across
 *                       step boundaries too); zl_comm_ll_begin_step(tp_comm) must be enqueued once per step before the
 *                       first such GEMM, on every rank.
 *   k_perm != NULL (act-order / desc_act GPTQ): y = W . x[:, k_perm], K int32 entries.  W is packed from the
 *                       sequentialised k-major tensors (zl_gptq_shuffle with q_perm = k_perm, the reference's
 *                       make_sequential, q_gemm.cu:794-829) and the activations are gathered while the integer kernel
 *                       stages them, where the reference runs permute_input first (gptq/utils.cu:322-398, called at
 *                       q_gemm_k_major.cu:1094, 1105).  ln_weight keeps the caller's (unpermuted) order: the prologue
 *                       uses x[k_perm[i]] * ln_weight[k_perm[i]]; the RMS is over the whole row, so the permutation does
 *                       not change it.  Only the exact-integer route (zl_w4_int_layout_route == 3) takes k_perm: the
 *                       wgmma and fp16 routes, and tp_mode != 0, return ZL_ERR_UNSUPPORTED (permute x with
 *                       zl_gather_cols_16 first).
 * bias is indexed by PACKED row. */
typedef struct zl_comm zl_comm_t;
typedef struct zl_w4_fused_args {
    const void* x; int ldx; const void* packed; const void* bias; const void* residual; void* y;
    int M, N, K, group_size, epilogue, pdl;
    const void* ln_weight; float eps;
    const float* cos; const float* sin; void* q_out;
    const int32_t* token_batch; const int32_t* placement; void* const* k_addrs; void* const* v_addrs;
    int num_heads, num_kv_heads, dim_head;
    const void* prefetch_ptr; size_t prefetch_bytes; /* next kernel's weights: pulled into L2 as this one drains (may be NULL) */
    int variant; /* layout of `packed`: 0 ZLW4, 1 ZLW4I (integer kernel; needs the staged activations to fit smem) */
    zl_comm_t* tp_comm; int tp_mode; void* tp_h_out; int tp_index;
    const int32_t* k_perm; /* act-order activation permutation (K), or NULL */
    /* int8 KV cache (ZL_EPI_QKV_ROPE on the exact-integer route only; the wgmma and fp16 routes and k_perm return
     * ZL_ERR_UNSUPPORTED): kv_int8 != 0 appends every K (after RoPE) / V row in the contract of zl_decode_attention_kv8 --
     * k_addrs / v_addrs are the tasks' uint8 code buffers, scale_k_addrs / scale_v_addrs their fp32 scale buffers -- with
     * the arithmetic of zl_kv_int8_quant_append, bit for bit.  kv8_stage: (M, 2, num_kv_heads, dim_head) fp16 scratch;
     * kv8_counters: (M, 2, num_kv_heads) uint32, zero before the first launch; each launch leaves them zero.  Launches that
     * share the counters must be stream-ordered. */
    int kv_int8; void* const* scale_k_addrs; void* const* scale_v_addrs; void* kv8_stage; uint32_t* kv8_counters;
} zl_w4_fused_args_t;
/* sizeof(zl_w4_fused_args_t) and offsetof(zl_w4_fused_args_t, k_perm), so that bindings can check their mirror. */
int zl_w4_fused_args_layout(size_t* size, size_t* k_perm_offset);
int zl_w4a16_gemm_fused(const zl_w4_fused_args_t* args, zl_stream_t stream);
/* 1 if the exact-integer kernel (variant 1, M <= 16) can run this shape: its staged activations must fit shared memory. */
int zl_w4_int_kernel_fits(int M, int N, int K);
/* which kernel serves (M, N, K) on the ZLW4I layout (variant 1): 3 = exact-integer mma.sync kernel, 4 = wgmma / TMA
 * kernel (any M, N % 128 == 0, no fused RMSNorm prologue), 0 = neither (pack variant 0 and use the fp16 mma.sync kernel). */
int zl_w4_int_layout_route(int M, int N, int K);
/* last watchdog code published by a tensor-core kernel on the current device (0 = none); a bounded mbarrier wait that expires
 * records which pipeline barrier starved and traps instead of hanging the GPU. */
unsigned zl_w4_tc_watchdog(void);
/* debug / tests: at least `splits` pieces per weight-row tile in the wgmma kernel's stream-k schedule (0 = automatic). */
int zl_w4_tc_set_splits(int splits);
/* tests: host view of the wgmma kernel's stream-k schedule (the kernel's own scheduling code): pieces of CTA `cta` of `ctas`
 * for n_tiles x G (tile, group) units; out[5 i ..] = tile, g0, g1, pieces of that tile, workspace slot (-1: whole tile);
 * returns the number of pieces. */
int zl_w4_tc_schedule(int n_tiles, int G, int ctas, int cta, int* out, int max_pieces);
/* host view of the variant the exact-integer kernel runs for (M <= 16 rows, N, K, tp_mode) on sm_count SMs: out[0..8] = NT,
 * warps per sub-CTA, sub-CTAs per CTA, ring stages, reduction rows, PACK, grid, dynamic shared memory bytes, sub-major tile
 * order (sub-CTA s of CTA b starts at tile s * grid + b instead of b * sub-CTAs + s); returns 0, or
 * ZL_ERR_UNSUPPORTED when none fits. */
int zl_w4_v3_plan(int mc, int N, int K, int tp_mode, int sm_count, int* out);
/* host view of the L2 head a predecessor GEMM prefetches for such a launch: the first H weight records each of its warps
 * requests, as out[3 i ..] = warp, byte offset, bytes; returns the number of ranges (<= max_ranges) or
 * a negative error code. */
int zl_w4_v3_l2_head(int mc, int N, int K, int tp_mode, int sm_count, int H, long long* out, int max_ranges);
/* debug: device buffer of grid*16 uint64 globaltimer samples written by the integer kernel (NULL = off). */
int zl_w4_set_trace(void* buf);
/* row_map (n_heads_total*dim_head) for zl_w4_pack so that RoPE partners (c, c+d/2) share an MMA tile. */
int zl_qkv_rope_row_map(int32_t* row_map, int n_heads_total, int dim_head, zl_stream_t stream);
/* dst[i] = src[map[i]] for 16-bit elements (bias permutation to packed-row order). */
int zl_gather_rows_16(const void* src, const int32_t* map, void* dst, int n, zl_stream_t stream);
/* y[m, i] = x[m, perm[i]] for 16-bit x (M, K) with row stride ldx and y (M, K) dense: the act-order activation permute
 * (nn::gptq::permute_input, gptq/utils.cu:322-398) for the GEMM routes that read x through TMA and cannot gather.
 * K % 8 == 0, ldx % 8 == 0, x and y 16-byte aligned.  pdl != 0 -> programmatic dependent launch. */
int zl_gather_cols_16(const void* x, int ldx, const int32_t* perm, void* y, int M, int K, int pdl, zl_stream_t stream);

/* ---- W8A8 Linear: SmoothQuant INT8 (Int8Linear, src/nn/linear/linear.cpp:432-636) and per-tensor FP8 e4m3
 * (Fp8Linear, linear.cpp:1612-1695) ---------------------------------------------------------------------- */
enum { ZL_W8_INT8 = 0, ZL_W8_FP8 = 1, ZL_W8_FP8_ROWS = 2 /* fp8 with one f32 weight scale per output row */ };
/* int8_op::quant_calc_scale (src/nn/quant/int8/quant_kernel.cu:15-103): per-token absmax quantisation,
 * scale[m] = absmax/127, q = int8(nearbyint(x * (127/absmax))).  x (M,K) f16/bf16 row stride ldx; q (M,K) int8. */
int zl_int8_quant_per_token(const void* x, int ldx, void* q, float* scale, int M, int K, int dtype, int pdl,
                            zl_stream_t stream);
/* int8_op::layernorm_quant (quant_kernel.cu:106-227): y = RMSNorm(x)*w/scale in T plus the int8 twin q with
 * qscale[t] = absmax(x*w) * rsqrt / 127. */
int zl_rmsnorm_quant(const void* x, const void* weight, void* y, void* q, float* qscale, int T, int D, float eps,
                     float scale, int dtype, int pdl, zl_stream_t stream);
/* nn::fp8::dynamic_scaled_quant (src/nn/quant/fp8/fp8_util.cu:110-228): *scale = absmax/448 over all n elements,
 * q = e4m3(sat(x * (1/scale))) with the reference's fp16 product rounding.  n <= 4 Mi elements (decode sizes). */
int zl_fp8_quant_per_tensor(const void* x, void* q, float* scale, size_t n, int dtype, int pdl, zl_stream_t stream);
/* Int8Linear::forward GEMM + int8_op::quant_scale_back (+add_bias), or Fp8Linear::forward's scaled fp8 GEMM, as ONE
 * kernel: y(M,N) = T(acc * x_scale * w_scale) (+bias).  xq (M,K) int8/e4m3; w (N,K) int8/e4m3 row-major (the
 * reference's parameter layout); kind ZL_W8_INT8: x_scale (M) f32, w_scale (N) of w_scale_dtype (ZL_F32 or dtype);
 * kind ZL_W8_FP8: both scales one f32.  INT8 results are bit-identical to the reference's three-kernel path. */
/* int8_op::quant_scale_back (quant_kernel.cu:231-306) stand-alone: y = T(float(acc) * x_scale[m] * w_scale[n]). */
int zl_int8_scale_back(const int32_t* acc, const float* x_scale, const void* w_scale, int w_scale_dtype, void* y, int M,
                       int N, int dtype, zl_stream_t stream);
int zl_w8a8_gemm(const void* xq, const float* x_scale, const void* w, const void* w_scale, int w_scale_dtype,
                 const void* bias, void* y, int M, int N, int K, int kind, int dtype, int pdl, zl_stream_t stream);

/* ---- FP8 block-scaled Linear (QuantType 10, Fp8Block, src/nn/linear/linear.cpp:1697-1960): e4m3 weights (N,K) with
 * one f32 weight_scale_inv per 128x128 block, activations quantised per token in groups of 128 along K ---------- */
/* nn::fp8::per_token_cast_to_fp8 (src/nn/quant/fp8/fp8_util.cu:231-322), bit for bit: per (token m, 128-column group kb)
 * amax = max(max|x|, 1e-4), q = e4m3(satfinite(x * (448/amax))) with the f32 product, scale[kb * scale_ld + m] =
 * amax/448 (column-major (K/128, scale_ld); the reference and DeepGEMM use scale_ld = round_up(M, 4)).
 * x (M,K) f16/bf16 with row stride ldx (ldx % 4 == 0, 8-byte aligned); q (M,K) e4m3 bytes.
 * K % 128 != 0 -> ZL_ERR_UNSUPPORTED. */
int zl_fp8_quant_per_token_group(const void* x, int ldx, void* q, float* scale, int scale_ld, int M, int K, int dtype,
                                 int pdl, zl_stream_t stream);
/* Fp8Block::forward's GEMM (deep_gemm_fp8_block_h20_group, linear.cpp:1697-1960) on the W8A8 kernels:
 * y[m,n] = T( sum_kb (sum_{k in kb} xq[m,k] * w[n,k]) * x_scale[kb * x_scale_ld + m] * w_scale[(n/128) * (K/128) + kb] ).
 * xq (M,K) e4m3 and w (N,K) e4m3 row-major, 16-byte aligned; x_scale as written by zl_fp8_quant_per_token_group;
 * w_scale (ceil(N/128), K/128) f32 row-major (N need not be a multiple of 128).  Output f16 or bf16, no bias.
 * mma.sync kernel up to M = 32, wgmma kernel in 256-row chunks above; each 128-k block's sum is promoted to f32 before
 * it is scaled.  K % 128 != 0 -> ZL_ERR_UNSUPPORTED. */
int zl_fp8_block_gemm(const void* xq, const float* x_scale, int x_scale_ld, const void* w, const float* w_scale, void* y,
                      int M, int N, int K, int dtype, int pdl, zl_stream_t stream);

/* functions::Gemm / NormalLinear for skinny M (lm_head, bf16 models; src/nn/linear/linear.cpp:150-430,
 * src/nn/embedding/embedding.cu:353-392): y(M,N) = x(M,K) @ W(N,K)^T (+bias), dtype f16/bf16,
 * out_dtype f16/bf16/f32. */
int zl_dense_gemm_skinny(const void* x, int ldx, const void* w, const void* bias, void* y, int M, int N, int K,
                         int dtype, int out_dtype, int pdl, zl_stream_t stream);

/* ------------------------------------------------------------------------------------------ *
 * Norm / residual / activation
 * ------------------------------------------------------------------------------------------ */
/* nn::LayerNorm::forward, rms (src/nn/layernorm/layernorm.cu:9-42): y = T(x*rsqrt(mean(x^2)+eps)*w/scale). */
int zl_rmsnorm(const void* x, const void* weight, void* y, int T, int D, float eps, float scale, int dtype,
               int pdl, zl_stream_t stream);
/* Residual + RMSNorm.  mode 0: block.cpp:124-131 order -- out_sum = T(a+b) (block_kernel.cu:7-17),
 * y = rmsnorm(out_sum);  mode 1: LayerNorm::fuse_add (layernorm.cu:28-41) -- y normalises the unrounded sum.
 * b may be NULL (then out_sum = a).  out_sum may alias a. */
int zl_add_rmsnorm(const void* a, const void* b, const void* weight, void* out_sum, void* y, int T, int D,
                   float eps, float scale, int mode, int dtype, int pdl, zl_stream_t stream);
/* nn::element_add_scale (src/nn/block/block_kernel.cu:7-17), scale_residual=false:
 * c = T(a + T(b*scale))  computed in T. */
int zl_element_add_scale(const void* a, const void* b, void* c, size_t n, float scale, int dtype,
                         zl_stream_t stream);
/* nn::gate_mul_inplace (src/nn/linear/activation_kernel.cu:55-106): out = T(act(float(gate))*float(up));
 * act 0 = silu, 1 = gelu.  gate/up (T, F) with row strides.  up == NULL: out = T(act(gate)), the activation
 * Linear::activate applies (src/nn/linear/linear.cpp activate(), activation_kernel.cu). */
int zl_gate_mul(const void* gate, int ld_gate, const void* up, int ld_up, void* out, int ld_out, int T, int F,
                int act, int dtype, zl_stream_t stream);

/* ------------------------------------------------------------------------------------------ *
 * RoPE + KV append
 * ------------------------------------------------------------------------------------------ */
/* RopePreparer (src/nn/position/rope_preparer.cu:49-161): cos/sin fp32 (T, d).
 * llama3_factor <= 0 -> plain rope. */
int zl_rope_cos_sin(const int32_t* pos, float* cos_out, float* sin_out, int T, int dim_head, float theta,
                    float llama3_factor, float low_freq_factor, float high_freq_factor, float old_context_len,
                    int neox, zl_stream_t stream);
/* nn::rope_qk_cache (src/nn/position/rotary_embedding_fuse_cache.cu:23-125): split fused qkv and rotate q,k. */
int zl_rope_qk_cache(const float* cos, const float* sin, const void* qkv, void* q, void* k, void* v, int T,
                     int num_heads, int num_kv_heads, int dim_head, int neox, int dtype, zl_stream_t stream);
/* nn copy_to_rag_buffer2 (src/kvcache/ragged_buffer_kernel.cu:194-300). */
int zl_copy_to_rag_buffer2(const int32_t* placement, const int32_t* buf_lens, const void* k_src,
                           const void* v_src, void* const* k_addrs, void* const* v_addrs, int B, int len_q,
                           int num_kv_heads, int dim_head, int bshd, int dtype, zl_stream_t stream);
/* Fused: split qkv (+bias already applied) + RoPE(q,k) + append K/V rows at placement into the per-task
 * buffers + write rotated q.  Replaces rope_qk_cache + copy_to_rag_buffer2 (attention.cpp:865-898, 636-676).
 * token_batch (T) int32: task index of each token; placement (T) int32 (<0: skip append). */
int zl_qkv_rope_append(const float* cos, const float* sin, const void* qkv, void* q_out,
                       const int32_t* token_batch, const int32_t* placement, void* const* k_addrs,
                       void* const* v_addrs, int T, int num_heads, int num_kv_heads, int dim_head, int neox,
                       int bshd, const int32_t* buf_lens, int dtype, int pdl, zl_stream_t stream);

/* ------------------------------------------------------------------------------------------ *
 * Decode attention over per-task ragged KV buffers
 * nn::multi_query_attention_rag_buffer (src/nn/attention/attention_kernel.cu:1252-1457)
 * ------------------------------------------------------------------------------------------ */
size_t zl_decode_attention_workspace_bytes(int B, int len_q, int num_heads, int dim_head, int max_len_buf);
/* q (B, len_q, H_q, d); buf_lens (B); k_addrs/v_addrs (B) device arrays of device pointers;
 * mask int8 ragged concat of (len_q, len_buf_b); out (B, len_q, H_q, d).  bshd: (len_buf, H_kv, d) else
 * (H_kv, len_buf, d). */
int zl_decode_attention(const void* q, const int32_t* buf_lens, void* const* k_addrs, void* const* v_addrs,
                        const int8_t* mask, float scale, int max_len_buf, void* out, int B, int len_q,
                        int num_heads, int num_kv_heads, int dim_head, int bshd, void* workspace,
                        size_t workspace_bytes, int dtype, int pdl, zl_stream_t stream);

/* Causal variable-length attention: every row of a joined chunked-prefill step (encode and search tokens of
 * SearcherImplV1::join_forward, src/generator/batch_generator.cpp:1337-1422, attended by Attention::dynamic_batch_forward,
 * src/nn/attention/attention.cpp:924-961, beam_size 1) in one launch, with no materialised mask.
 * seg (nseg, 4) int32 DEVICE array, 16-byte aligned, of segments {task, row0, pos0, n}: rows row0 .. row0 + n - 1 of q
 * hold positions pos0 .. pos0 + n - 1 of task `task`, and the row at position p attends keys 0 ..= p of that task's cache.
 * A decode row is a segment with n = 1.  q / out (rows, H_q, d); k_addrs / v_addrs per-task BSHD caches (len, H_kv, d)
 * as for zl_decode_attention; every segment needs pos0 + n <= max_keys; keys past a row's position are never read.
 * fp16 / bf16, d = 64 or 128, H_q % H_kv == 0.  Splits cover fixed 512-key ranges, so a row's output bits depend only on
 * its q, its task's cache and its position, not on the other segments.  workspace: zl_varlen_attention_workspace_bytes
 * (0 when max_keys <= 512). */
size_t zl_varlen_attention_workspace_bytes(int rows, int nseg, int num_heads, int dim_head, int max_keys);
int zl_varlen_attention(const void* q, const int32_t* seg, int nseg, int rows, void* const* k_addrs, void* const* v_addrs,
                        float scale, int max_keys, void* out, int num_heads, int num_kv_heads, int dim_head, void* ws,
                        size_t ws_bytes, int dtype, int pdl, zl_stream_t stream);

/* MLA decode attention over per-task latent caches: nn::multi_query_attention_rag_buffer with dim_head 576 and a
 * 512-wide output, as the reference's MLA search path calls it (src/nn/attention/multi_head_latent_attention.cpp:1053-1068;
 * kernels attention_kernel.cu:1281-1284, 1347-1348, 1390-1391, 1429-1435), and the per-task GEMM / softmax / GEMM of its
 * attn_by_gemm (multi_head_latent_attention.cpp:834-874).
 * q (B, len_q, H, 576); kv_addrs (B) device array of device pointers, task b's latent rows (len_buf_b, 576): the first 512
 * elements of a row are its value, the whole row its key, shared by all H heads; buf_lens (B); mask optional int8 ragged
 * concat of (len_q, len_buf_b) as for zl_decode_attention; out (B, len_q, H, 512).  Row (b, i, h) attends keys
 * 0 .. buf_lens[b] - 1: logit = mask ? scale * q.k : -inf, o = softmax . v (max seeded -1e20, sum seeded 1e-20), so a row
 * with every key masked gives 0.  Rows past buf_lens[b] are never read.  fp16 / bf16, 1 <= H <= 128 (ZL_ERR_UNSUPPORTED
 * above).  workspace: at least zl_mla_decode_attention_workspace_bytes (0 when max_len_buf <= 256); two launches give
 * bit-identical output. */
size_t zl_mla_decode_attention_workspace_bytes(int B, int len_q, int num_heads, int max_len_buf);
int zl_mla_decode_attention(const void* q, const int32_t* buf_lens, void* const* kv_addrs, const int8_t* mask,
                            float scale, int max_len_buf, void* out, int B, int len_q, int num_heads,
                            void* workspace, size_t workspace_bytes, int dtype, int pdl, zl_stream_t stream);

/* int8 KV cache (KV_CACHE_DTYPE=int8 of the reference): KERNEL_mqa_rag_buffer_split_kv_quant
 * (src/nn/attention/attention_kernel.cu:804-880, src/nn/attention/quant_attention.cuh:10-123).  K / V buffers per task are
 * (len_buf, H_kv, d) uint8 = round(x * 127 / absmax) + 128, scale buffers (len_buf, H_kv) fp32 = absmax / 127 (BSHD only,
 * like the reference); q is fp16; out in out_dtype.  Any max_len_buf (the reference only takes this path above
 * ATTN_SPLIT_KV_THRES = 1024).  workspace as zl_decode_attention_workspace_bytes. */
int zl_decode_attention_kv8(const void* q, const int32_t* buf_lens, void* const* k_addrs, void* const* v_addrs,
                            void* const* scale_k_addrs, void* const* scale_v_addrs, const int8_t* mask, float scale,
                            int max_len_buf, void* out, int B, int len_q, int num_heads, int num_kv_heads, int dim_head,
                            void* workspace, size_t workspace_bytes, int out_dtype, int pdl, zl_stream_t stream);
/* cache side of the same contract: int8_op::quant_calc_scale(x, 127, 128) per (token, kv head) row
 * (src/nn/quant/int8/quant_kernel.cu:15-47) + copy_to_rag_buffer2 of the codes and of the scales
 * (src/nn/attention/attention.cpp:656-676): k_src / v_src (T, H_kv, d), token t goes to row placement[t] of task
 * token_batch[t] (placement < 0: skipped). */
/* the same quantisation on dense rows: x (M, K) -> q (M, K) uint8, scale (M) fp32 (quant_calc_scale(x, 127, 128)). */
int zl_int8_quant_rows_u8(const void* x, void* q, float* scale, int M, int K, int dtype, zl_stream_t stream);
int zl_kv_int8_quant_append(const void* k_src, const void* v_src, const int32_t* token_batch, const int32_t* placement,
                            void* const* k_addrs, void* const* v_addrs, void* const* scale_k_addrs,
                            void* const* scale_v_addrs, int T, int num_kv_heads, int dim_head, int dtype, int pdl,
                            zl_stream_t stream);

/* ------------------------------------------------------------------------------------------ *
 * Decode-step helpers around the layers
 * ------------------------------------------------------------------------------------------ */
/* nn::Embedding lookup (src/nn/embedding/embedding.cu:20-60): out[t,:] = table[ids[t],:]. */
int zl_embedding(const int32_t* ids, const void* table, void* out, int T, int D, int vocab, int dtype, int pdl,
                 zl_stream_t stream);
/* greedy pick (generator/batch_generator.cpp:1762-1884 with beam 1): argmax over fp32 logits (T, V). */
size_t zl_argmax_workspace_bytes(int T);
int zl_argmax(const float* logits, int32_t* out, int T, int V, void* workspace, size_t workspace_bytes, int pdl,
              zl_stream_t stream);
/* vocab-parallel pick: per-token {float value, int global index} candidate of one logits shard (T, V), and the
 * merge over the all-gathered candidates [ranks][stride] (embedding.cu:353-392 gathers the logits instead). */
int zl_argmax_candidates(const float* logits, void* cand_out, int T, int V, int idx_offset, void* workspace,
                         size_t workspace_bytes, int pdl, zl_stream_t stream);
int zl_argmax_merge(const void* cand_all, int32_t* out, int T, int ranks, int stride, int pdl, zl_stream_t stream);

/* Next-token sampling (SearcherImplV1::random_sample, generator/batch_generator.cpp:1854-1883 = functions::softmax with
 * temperature (softmax.cu) + beam_utility::random_sampler_gpu (generator/random_util.cu:81-198), with the penalties of
 * beam_repetition_penalty (generator/beam_util.cu:198-281)).  Per task:
 *   temperature >= 0, top_p in (0, 1], top_k >= 0 (0 or >= V: off), repetition_penalty > 0, presence_penalty, seed.
 * A row's token depends only on its fp32 logits, its task's parameters and seed, its counter and its task's history:
 *   1. penalties, on a copy of the logits, for every token set in the task's history bitmap (the distinct tokens
 *      generated since the task's sampling was last set): presence_penalty != 0 ? l -= presence_penalty
 *      : l = l < 0 ? l * repetition_penalty : l / repetition_penalty   (beam_util.cu:212-219);
 *   2. temperature == 0 or top_k == 1: greedy, exactly zl_argmax's pick of the penalised row (ties -> lowest index);
 *   3. otherwise x = l / temperature in descending order (ties by ascending index), w = exp(x - max x), Z = sum w,
 *      C_j the inclusive cumulative sum in that order, P' = min(top_p * Z, C_{top_k-1}) (Z when top_k is off),
 *      target = u * P'; the token is the first j with C_j >= target  (random_util.cu:89-106);
 *   4. u = ((r >> 8) + 1) * 2^-24 with r = zl_sample_uniform(seed, counter);
 *   5. -inf / NaN logits have probability 0; a row whose penalised max is not finite takes the greedy pick.
 * Masses are summed as exact 2^-44 fixed-point integers (deterministic; a token below ~2^-45 of the row's maximum weight
 * has probability 0).  After the pick the token's bit is set in the task's history.
 * Whether to sample is the scheduler's decision: the reference samples only when top_p < 1 or top_k > 0
 * (SearchTask::is_random, batch_generator.h:106); a scheduler maps is_random() == false to temperature = 0. */
typedef struct zl_sample_params {
    float temperature, top_p, repetition_penalty, presence_penalty;
    int top_k;
    uint64_t seed;
} zl_sample_params_t;
/* r: the first 32-bit output of Philox4x32-10 (curand_philox4x32_x.h round function and constants) with
 * key = (seed low, seed high) and counter = (counter, 0, 0, 0).  The kernel draws the same r on the device. */
unsigned zl_sample_uniform(uint64_t seed, unsigned counter);
/* host check of n parameter sets (HOST pointer): ZL_ERR_INVALID_ARG for values outside the ranges above. */
int zl_sample_check_params(const zl_sample_params_t* params_host, int n);
/* 0 today: the sampler keeps everything in shared memory (ws may be NULL). */
size_t zl_sample_workspace_bytes(int T, int V);
/* logits (T, V) fp32; params indexed by task; row_task (T) maps rows to tasks (NULL: row i is task i); counter (T) the
 * position of the input token whose logits each row holds (NULL: 0); history (tasks, history_words >= ceil(V/32)) u32
 * bitmap or NULL (no penalties, nothing recorded; rows sharing a task must not pass a history); out (T) int32.
 * V <= 262144 (ZL_ERR_UNSUPPORTED above).  One launch: one cluster of 8 CTAs per row.  Parameter values are not
 * checked on the device: validate them with zl_sample_check_params. */
int zl_sample(const float* logits, int T, int V, const zl_sample_params_t* params, const int32_t* row_task,
              const int32_t* counter, uint32_t* history, int history_words, int32_t* out, void* ws, size_t ws_bytes,
              int pdl, zl_stream_t stream);
/* Logits processors on top of zl_sample: the n-gram repetition penalty (calc_repetition_ngram +
 * apply_beam_repetition_penalty, generator/beam_util.cu:318-375, chosen at batch_generator.cpp:1662-1705) and logit_bias
 * (SearcherImplV1::add_logit_bias, batch_generator.cpp:1709-1728).  For a row of task t, on a copy of its fp32 logits:
 *   1. penalties.  ngram_penalty[t] > 1: with r the task's sequence most recent first and lev[j] the reference's
 *      ngrams[j] of r (KMP next[] over r, then ngrams[i - L] = max(ngrams[i - L], L) with L = next[i] + 1), every token
 *      occurring in r gets f = max over its occurrences j of powf(ngram_penalty, lev[j] + 1) * repetition_penalty and
 *      l = l < 0 ? l * f : l / f; presence_penalty is ignored (the reference's n-gram path passes no presence values).
 *      Otherwise (ngram_penalty NULL or <= 1) zl_sample's bitmap rule, unchanged;
 *   2. l += bias for each (token, bias) entry of the task, in fp32 (the reference adds it in the logits dtype);
 *   3. the pick: steps 2-5 of zl_sample's contract on the processed row.
 * The rule is chosen per task, so a row's token depends only on its logits, its task's parameters, bias list and
 * sequence, and its counter; never on the batch (the reference decides the n-gram path per batch).
 * ngram_penalty (tasks) fp32 or NULL (no n-gram launch); seq (tasks, seq_stride) int32 generated tokens, oldest first, with
 * seq_len (tasks): the pick is appended there (dropped once seq_len == seq_stride), as zl_sample records it into history;
 * rows naming one task must not pass a sequence.  bias_tokens / bias_values (tasks, bias_stride) with bias_count (tasks),
 * or NULL: distinct tokens per task (a repeated token is added once per entry; ids outside [0, V) are ignored).
 * ws: zl_sample_processed_workspace_bytes(T, seq_stride) bytes when ngram_penalty is given (k_ngram_levels writes each
 * row's distinct tokens and levels there), else may be NULL.  Launches: k_sample, plus k_ngram_levels (one CTA per row;
 * rows whose task has ngram_penalty <= 1 exit at once) when ngram_penalty is given. */
#define ZL_MAX_LOGIT_BIAS 1024
size_t zl_sample_processed_workspace_bytes(int T, int seq_stride);
int zl_sample_processed(const float* logits, int T, int V, const zl_sample_params_t* params, const int32_t* row_task,
                        const int32_t* counter, uint32_t* history, int history_words, const float* ngram_penalty,
                        int32_t* seq, int32_t* seq_len, int seq_stride, const int32_t* bias_tokens,
                        const float* bias_values, const int32_t* bias_count, int bias_stride, int32_t* out, void* ws,
                        size_t ws_bytes, int pdl, zl_stream_t stream);
/* Allowed-token masks on top of zl_sample_processed (structured output: a token automaton's allowed set, or a grammar
 * engine's per-step bitmask).  masks (rows, mask_words >= ceil(V/32)) u32: bit j of word i allows token 32 i + j.
 * mask_row (tasks) int32 or NULL: task t is masked by row mask_row[t] (< rows, not checked on the device), or not at all
 * when mask_row[t] < 0; NULL masks task t by row t.  For a masked row, with A its allowed set:
 *   0. every token outside A is removed before anything else: it is never picked, gets no mass and does not count for
 *      top_k (as a NaN logit); an allowed NaN logit counts as -inf;
 *   1.-3. zl_sample_processed's contract, unchanged, on the tokens of A: penalties, n-gram rule, bias, temperature, top-k,
 *      top-p and the Philox draw; greedy rows (temperature 0 or top_k 1) take the lowest-index maximum over A;
 *   4. when every token of A ends at -inf after the bias, the pick is the smallest token of A.
 * A is expected non-empty (an empty row picks token 0).  Unmasked rows get exactly zl_sample_processed's token. */
int zl_sample_masked(const float* logits, int T, int V, const zl_sample_params_t* params, const int32_t* row_task,
                     const int32_t* counter, uint32_t* history, int history_words, const float* ngram_penalty,
                     int32_t* seq, int32_t* seq_len, int seq_stride, const int32_t* bias_tokens, const float* bias_values,
                     const int32_t* bias_count, int bias_stride, const uint32_t* masks, int mask_words,
                     const int32_t* mask_row, int32_t* out, void* ws, size_t ws_bytes, int pdl, zl_stream_t stream);
/* Beam-search selection (beam_utility::log_softmax_bias, generator/beam_util.cu:20-130, then topk_all.get_top_k over each
 * task's flattened (beam x vocab) scores, generator/batch_generator.cpp:1770-1778), without writing an (R, V) tensor.
 * logits (R, V) fp32 and cum (R) fp32 on the device; groups (G, 2) {row0, width} a HOST array whose groups tile rows
 * [0, R) in order.  For each group g the K largest s = cum[r] + logits[r, v] - lse_r over its rows r and every v, with
 * lse_r = max_r + log(1e-20 + sum_v exp(logits[r, v] - max_r)) in fp32, sorted by score descending and ties by the flat
 * index (r - row0) * V + v ascending: parent[g, k] = r - row0, token[g, k] = v, score[g, k] = s (device (G, K) arrays).
 * A row with cum = -inf is dead: its logits are never read (they may hold NaN).  Only finite scores are candidates; a group
 * with fewer than K gets parent = token = -1 and score = -inf in the rest.  1 <= K <= 32 and 1 <= width <= 16, else
 * ZL_ERR_INVALID_ARG; V > 262144: ZL_ERR_UNSUPPORTED; every check runs before anything is enqueued.  Two launches, after
 * a copy of the groups into the workspace (ws_bytes >= zl_beam_topk_workspace_bytes(R, V, K)). */
size_t zl_beam_topk_workspace_bytes(int R, int V, int K);
int zl_beam_topk(const float* logits, int R, int V, const float* cum, const int32_t* groups, int G, int K,
                 int32_t* parent, int32_t* token, float* score, void* ws, size_t ws_bytes, int pdl, zl_stream_t stream);
/* synthetic-checkpoint generators (bench / tests): counter-based hash RNG, reproducible per seed. */
int zl_fill_random_u32(uint32_t* p, size_t n, uint64_t seed, zl_stream_t stream);
int zl_fill_const_u32(uint32_t* p, size_t n, uint32_t value, zl_stream_t stream);
int zl_fill_uniform(void* p, size_t n, float lo, float hi, uint64_t seed, int dtype, zl_stream_t stream);

/* ------------------------------------------------------------------------------------------ *
 * Tensor-parallel exchange over NVLink peer memory (one process per GPU, one node)
 * Replaces ModelContext::reduce_sum / reduce_sum2 / reduce_tp_int8 (src/model/model_context.cpp:203-326) and
 * the c10d NCCL wrappers it calls (3rd/bmengine/bmengine/c10d/c10d.cpp:42-136) on the decode path.
 * ------------------------------------------------------------------------------------------ */
/* Allocates this rank's symmetric buffer (inboxes for world_size sources x 2 parities of max_elems 16-bit values). */
int zl_comm_create(int rank, int world_size, size_t max_elems_16bit, zl_comm_t** out);
void zl_comm_destroy(zl_comm_t* c);
int zl_comm_rank(zl_comm_t* c);
int zl_comm_world_size(zl_comm_t* c);
/* CUDA IPC handle of the symmetric buffer (zl_comm_ipc_handle_bytes() bytes); exchange them out of band
 * (torch.distributed all_gather in zhilight_b200/dist.py) and hand all of them (index = rank) to open_peers. */
int zl_comm_ipc_handle_bytes(void);
int zl_comm_get_ipc_handle(zl_comm_t* c, void* handle_out);
int zl_comm_open_peers(zl_comm_t* c, const void* handles_all);
/* once per decode step that uses the exchange fused into the W4 GEMMs (tp_mode of zl_w4a16_gemm_fused), before the first
 * such GEMM of the step and on every rank: advances the step counter the word tags are derived from. */
int zl_comm_ll_begin_step(zl_comm_t* c, zl_stream_t stream);
/* tests: this rank's symmetric buffer (device pointer) and its size in bytes. */
int zl_comm_local_buffer(zl_comm_t* c, void** base, size_t* bytes);
/* out = T(T(sum over ranks of partial) + residual); n % 32 == 0; residual may be NULL; out may alias residual.
 * int8_payload != 0: peers' contributions travel as int8 + one T scale per 32 values (the reference's group-32
 * format, int8/quant_reduce_kernel.cu:14-38); deterministic rank-ordered fp32 reduction either way. */
int zl_allreduce_one_shot(zl_comm_t* c, const void* partial, const void* residual, void* out, size_t n, int dtype,
                          int int8_payload, int pdl, zl_stream_t stream);
/* out[r*bytes ..] = `in` of rank r (bytes % 16 == 0, small: one CTA). */
int zl_allgather_small(zl_comm_t* c, const void* in, void* out, size_t bytes, int pdl, zl_stream_t stream);
/* Vocabulary all-gather for the full-vocabulary picks under tensor parallelism (the NCCLAllGather of the logit shards in
 * src/nn/embedding/embedding.cu:353-390).  Each rank owns a (max_rows, vocab) fp32 row-major buffer, mapped into the
 * peers with CUDA IPC like zl_comm's (handles of zl_comm_ipc_handle_bytes() bytes, index = rank); world_size 1 needs no
 * peers.  zl_vocab_allgather writes rows 0 .. rows-1 of this rank's (rows, vocab / world_size) shard (row stride ld floats,
 * 16-byte aligned) into columns [rank * vshard, (rank + 1) * vshard) of every rank's buffer, this one's included, and
 * returns on the device once every rank's shard has arrived here: one launch, a collective that every rank must enqueue
 * with the same rows.  A rank's next gather may overwrite the buffer as soon as every rank has enqueued its own, so a
 * reader must finish before an exchange that all ranks reach before their next gather (the decode driver's all-reduces).
 * create: vocab % world_size != 0, max_rows < 1 or max_rows * vocab >= 2^31: ZL_ERR_INVALID_ARG; (vocab / world_size) % 4
 * != 0: ZL_ERR_UNSUPPORTED.  gather: rows outside [1, max_rows], ld < vshard, ld % 4 != 0 or a misaligned shard:
 * ZL_ERR_INVALID_ARG; peers not opened: ZL_ERR_STATE; nothing is enqueued then. */
typedef struct zl_vocab_gather zl_vocab_gather_t;
int zl_vocab_gather_create(int rank, int world_size, int max_rows, int vocab, zl_vocab_gather_t** out);
void zl_vocab_gather_destroy(zl_vocab_gather_t* g);
int zl_vocab_gather_get_ipc_handle(zl_vocab_gather_t* g, void* handle_out);
int zl_vocab_gather_open_peers(zl_vocab_gather_t* g, const void* handles_all);
int zl_vocab_gather_info(zl_vocab_gather_t* g, int* rank, int* world_size, int* max_rows, int* vocab);
/* the (max_rows, vocab) buffer of this rank (device pointer; NULL for g == NULL) */
float* zl_vocab_gather_buffer(zl_vocab_gather_t* g);
int zl_vocab_allgather(zl_vocab_gather_t* g, const float* shard, int rows, int ld, int pdl, zl_stream_t stream);
/* int8_op::quant_group_32 / dequant_sum_quant_g32 / dequant_group_32 / dequant_group_fuse_add
 * (src/nn/quant/int8/quant_reduce_kernel.cu:14-38, 243-322, 105-140, 201-240); M = number of 32-groups. */
int zl_quant_group_32(const void* in, int8_t* out_q, void* out_scale, size_t M, int dtype, zl_stream_t stream);
int zl_dequant_sum_quant_g32(const void* my, const int8_t* q_others, const void* scale_others, int8_t* out_q,
                             void* out_scale, size_t M, int world_size, int dtype, zl_stream_t stream);
/* add != NULL: dequant_group_fuse_add (out = q*s + add). */
int zl_dequant_group_32(const int8_t* q, const void* scale, const void* add, void* out, size_t M, int dtype,
                        zl_stream_t stream);

/* ------------------------------------------------------------------------------------------ *
 * Decode driver: the model::LLaMA::encode + get_logits + greedy pick stand-in
 * (src/model/llama.cpp:75-165, src/nn/block/block.cpp:86-143, src/nn/attention/attention.cpp:846-964,
 *  src/nn/feedforward/feedforward.cpp:113-137) for len_q = 1 dynamic-batch steps.  The reference keeps
 * its scheduler (src/generator) above this; here the caller supplies (token, position) per task.
 * One CUDA graph per batch size, all kernels chained with programmatic dependent launch.
 * ------------------------------------------------------------------------------------------ */
typedef struct zl_llama zl_llama_t;
typedef struct zl_llama_config {
    int num_layers, dim_model, num_heads, num_kv_heads, dim_head, dim_ff, vocab_size;
    float eps, rope_theta;
    float rope_llama3_factor; /* <= 0: plain rope */
    float rope_low_freq_factor, rope_high_freq_factor, rope_orig_ctx;
    int quant_type; /* model_config.hpp:132-144 QuantType: 0 none, 2 AutoInt8 (fp weights quantised per row at load),
                     * 5 GPTQ, 6 AWQ, 7 FP8 (e4m3 weights + per-tensor weight_scale), 8 GPTQ_Marlin (= 5 with sym),
                     * 10 FP8_Block (e4m3 weights + weight_scale_inv (ceil(N/128), K/128) f32; tp_size 1, no qkv_bias,
                     * dim_model, q/k/v widths and dim_ff multiples of 128, else ZL_ERR_UNSUPPORTED) */
    int group_size, sym;
    int dtype; /* ZL_F16 / ZL_BF16 (W4 paths are fp16-only like the reference, q_gemm_k_major.cu:989) */
    int max_batch, max_seq;
    int tp_rank, tp_size;
    int use_pdl, use_graph;
    int tp_int8; /* TP all-reduce payload: 0 = activation dtype, 1 = int8 group-32 (REDUCE_TP_INT8 of the reference) */
    int fuse; /* 0: one kernel per reference operator; 1: RMSNorm folded into the W4 GEMMs; 2 (3 is accepted as 2):
               * + qkv RoPE/KV-append epilogue.  Launches with more than 16 tokens run zl_rmsnorm + the wgmma GEMM. */
    int prefill_chunk; /* 0: decode only.  1..2048: zl_llama_prefill processes a prompt in chunks of this many tokens
                        * (chunked prefill, zhilight/config/adapter.py:47-48) */
    int qkv_bias; /* zl_llama_init_synthetic: also create q/k/v biases (Qwen2: attention.cpp:105-109); loaded checkpoints
                   * carry their ".bias" tensors regardless of this flag */
    int kv_int8; /* 0: KV cache in the activation dtype.  1: int8 KV cache (KV_CACHE_DTYPE=int8, model_context.cpp:61-79) in
                  * the contract of zl_decode_attention_kv8: every appended K (after RoPE) / V row is quantised per
                  * (token, kv head) and decode, chunked prefill and the dual-stream prefill attend over the quantised
                  * cache with zl_decode_attention_kv8 (the reference attends a prompt over an fp16 copy of its own K/V).
                  * fp16 only, dim_head 64 or 128, max_seq <= 65536: other configurations return ZL_ERR_UNSUPPORTED */
    int kv_rows; /* 0: fixed KV layout, task t owns rows [t max_seq, (t + 1) max_seq) of every layer for good.  1 ..
                  * max_batch * max_seq (else ZL_ERR_INVALID_ARG): a KV arena of this many rows per layer (rounded up to
                  * 64), shared by every task slot.  Tasks start with no rows; before a call writes rows up to r of a task,
                  * the task is granted at least r + 1 (geometric growth, a move or a compaction of the other tasks, the new
                  * rows zero-filled).  Each entry point that writes rows returns ZL_ERR_KV_FULL when they cannot be
                  * granted.  zl_llama_kv_release returns a task's rows. */
} zl_llama_config_t;
/* sizeof(zl_llama_config_t) and offsetof(zl_llama_config_t, kv_int8), so that bindings can check their mirror. */
int zl_llama_config_layout(size_t* size, size_t* kv_int8_offset);

int zl_llama_create(const zl_llama_config_t* cfg, zl_llama_t** out);
/* tensor parallel: hand the driver its exchange object (zl_comm_create + open_peers) before the first step. */
int zl_llama_set_comm(zl_llama_t* m, zl_comm_t* comm);
/* tensor parallel: serve the full-vocabulary picks -- sampling, logits processors, beam steps and zl_llama_generate -- by
 * gathering the lm_head shards into g (zl_vocab_gather_create with this rank and world size, max_rows >= max_batch,
 * vocab == vocab_size, peers opened) before the sampler or zl_beam_topk, which then run on every rank over the same rows
 * and pick the same tokens.  Greedy-only steps keep the candidate exchange.  Without it those entry points return
 * ZL_ERR_UNSUPPORTED under tp_size > 1.  Every rank must make the same zl_llama_set_sampling, set_logits_processors,
 * set_stop, beam_step and generate calls, as they make the same set_state and decode calls: ranks that disagree on
 * whether a step samples wait on different exchanges.  g must outlive the model's steps.  Mismatched g:
 * ZL_ERR_INVALID_ARG. */
int zl_llama_set_vocab_gather(zl_llama_t* m, zl_vocab_gather_t* g);
void zl_llama_destroy(zl_llama_t* m);
/* Stage one checkpoint tensor (HOST pointer, row-major (rows, cols)); names as produced by
 * zhilight/loader.py:250-358 without the "llama." prefix, e.g. "layers.0.attn.project_q.qweight". */
int zl_llama_load_tensor(zl_llama_t* m, const char* name, const void* data_host, int rows, int cols,
                         int elem_bytes);
/* Fill every tensor of the configured architecture with reproducible random data ON DEVICE
 * (HF-GPTQ layout for quantized linears) and run the load pipeline layer by layer. */
int zl_llama_init_synthetic(zl_llama_t* m, uint64_t seed);
/* Run the load pipeline (Int4GPTQ::preprocess_weight + fusion + ZLW4 pack) on the staged tensors. */
int zl_llama_finalize(zl_llama_t* m);
/* One decode step for B tasks.  tokens_host/positions_host (B) int32; task b owns KV slot b.
 * next_tokens_host (B) int32 greedy picks; logits_host NULL or (B, vocab) fp32.  Synchronous.
 * KV arena: ZL_ERR_KV_FULL when a task's row at its position cannot be granted (also zl_llama_step_device). */
int zl_llama_decode(zl_llama_t* m, const int32_t* tokens_host, const int32_t* positions_host, int B,
                    int32_t* next_tokens_host, float* logits_host);
/* Device-resident variant: stage tokens/positions once, then each call replays the step, feeds the picked
 * tokens back and advances positions on the device; no host sync.  The host mirrors the positions, so a KV arena grants
 * each step's rows before the step is enqueued (ZL_ERR_KV_FULL when it cannot). */
int zl_llama_set_state(zl_llama_t* m, const int32_t* tokens_host, const int32_t* positions_host, int B);
int zl_llama_step_device(zl_llama_t* m, int B);
/* read back the device-resident (token, position) state; synchronous. */
int zl_llama_get_state(zl_llama_t* m, int32_t* tokens_host, int32_t* positions_host, int B);
/* fp32 logits (B, vocab/tp) of the last step (device-resident or host-API), this rank's vocabulary shard.  Synchronous. */
int zl_llama_get_logits(zl_llama_t* m, float* logits_host, int B);
int zl_llama_sync(zl_llama_t* m);
/* Chunked prefill of ONE task (SearchTask prompt, src/generator/batch_generator.cpp:1576): appends tokens_host[0..n) at
 * positions pos0.. to the task's KV buffers through the same kernels (M = chunk GEMMs, causal len_q = chunk attention)
 * and returns the greedy next token (and optionally the last position's logits, vocab/tp floats).  Synchronous.
 * KV arena: rows up to pos0 + n are granted before the first chunk, or ZL_ERR_KV_FULL with nothing enqueued. */
/* Prefill keeps its own token / position staging on the device: the (token, position) state of the decode tasks set by
 * zl_llama_set_state survives a prefill issued between two zl_llama_step_device calls (continuous batching).  It
 * overwrites the next-token / logits row 0 outputs, which zl_llama_step_device consumes before it returns. */
int zl_llama_prefill(zl_llama_t* m, int task, const int32_t* tokens_host, int n, int pos0, int32_t* next_token_host,
                     float* logits_host);
/* One forward over nseg segments, the joined step of chunked-prefill scheduling (SearcherImplV1::join_forward,
 * src/generator/batch_generator.cpp:1337-1422): prompt chunks and decode rows of different tasks stream the weights once.
 * seg_host (nseg x 4, HOST) = {task, pos0, n, emit}; tokens_host = the segments' tokens concatenated.  Rows sum(n) <=
 * max(max_batch, prefill_chunk); distinct tasks; pos0 + n <= max_seq.  Each segment appends its n K/V rows at pos0.. of its
 * task and attends causally (zl_varlen_attention).  For each segment with emit != 0 its LAST row goes through the final
 * norm, lm_head and the pick (greedy, or per-task sampling with counter = that row's position, recorded in the task's
 * history); next_host (nseg) gets the pick or -1, logits_host (n_emit x vocab, segment order) may be NULL.  The
 * device-resident decode state (zl_llama_set_state) survives the call, as it survives a prefill.  Synchronous, no graph.
 * prefill_chunk == 0: ZL_ERR_STATE; malformed segments: ZL_ERR_INVALID_ARG; kv_int8 or tp_size > 1: ZL_ERR_UNSUPPORTED;
 * a KV arena that cannot grant every segment's rows: ZL_ERR_KV_FULL. */
int zl_llama_step_joined(zl_llama_t* m, const int32_t* tokens_host, const int32_t* seg_host, int nseg, int32_t* next_host,
                         float* logits_host);
/* Per-task sampling (zl_sample's contract) for the picks of zl_llama_decode / step_device / prefill.  Copies *p (HOST
 * pointer) to the device and clears the task's history and generated-token sequence; p == NULL returns the task to plain greedy.  Invalid values:
 * ZL_ERR_INVALID_ARG; anything but plain greedy under tp_size > 1 without zl_llama_set_vocab_gather: ZL_ERR_UNSUPPORTED
 * (vocabulary shards would need a global top-k / top-p threshold).  The decode step runs zl_sample instead of zl_argmax while a task in the batch
 * samples or has penalties (counter = the input token's position; prefill: pos0 + n - 1), so a task draws the same
 * tokens with host or device-resident stepping, with or without the graph.  The logits stay the raw lm_head output. */
int zl_llama_set_sampling(zl_llama_t* m, int task, const zl_sample_params_t* p);
/* Per-task logits processors (zl_sample_processed's contract) for the picks of zl_llama_decode / step_device / prefill /
 * step_joined.  Stream-ordered after the steps already enqueued; the HOST arrays are staged before the call returns.
 * ngram_penalty finite and > 0 (<= 1: off, batch_generator.cpp:1664); n_bias in [0, ZL_MAX_LOGIT_BIAS] distinct tokens in
 * [0, vocab) with finite or -inf values (NaN and +inf are refused): ZL_ERR_INVALID_ARG otherwise.  n_bias = 0 with
 * ngram_penalty <= 1 returns the task to plain behaviour.  Anything on under tp_size > 1 without zl_llama_set_vocab_gather:
 * ZL_ERR_UNSUPPORTED.  Every
 * check runs before anything is enqueued.  A task with processors makes its batch's pick run the sampler, as a penalty
 * does.  The n-gram rule reads the task's generated-token sequence: the picks of the sampler route since
 * zl_llama_set_sampling last cleared it, up to max_seq tokens (later picks are not recorded). */
int zl_llama_set_logits_processors(zl_llama_t* m, int task, float ngram_penalty, const int32_t* bias_tokens_host,
                                   const float* bias_values_host, int n_bias);
/* Constrained decoding: a per-task token automaton whose state's allowed set masks the task's picks (zl_sample_masked's
 * contract) and whose state moves on the device with every recorded pick.  An automaton has S >= 1 states; state s has
 * a non-empty allowed set A(s), ceil(vocab/32) u32 words with no bit at or past vocab (bit j of word i = token 32 i + j),
 * edges (token, next) with distinct tokens of A(s) in ascending order, and default_next[s].  Picking x in state s moves
 * the task to the next state of x's edge, or to default_next[s] when x has none.  The state moves exactly where a pick is
 * recorded: zl_llama_decode / step_device rows, the last chunk of zl_llama_prefill, the emitting segments of
 * zl_llama_step_joined and the running tasks of zl_llama_generate (a finished task neither records nor moves).  The
 * returned logits stay raw.  A one-state automaton whose default is itself is a plain mask; setting one before each
 * zl_llama_decode is how a host grammar engine drives the engine step by step.
 * zl_llama_enable_constraints allocates, per task, max_states masks, max_states + 1 row offsets, max_edges edges and
 * max_states defaults on the device, once per model (a second call: ZL_ERR_STATE; before zl_llama_finalize:
 * ZL_ERR_STATE; max_states < 1 or max_edges < 0: ZL_ERR_INVALID_ARG).  Graphs captured before it are dropped. */
int zl_llama_enable_constraints(zl_llama_t* m, int max_states, int max_edges);
/* Host check of one automaton over a vocabulary of `vocab` tokens (HOST arrays, as zl_llama_set_constraint takes them,
 * n_states >= 1): ZL_ERR_INVALID_ARG for every malformation listed there, else ZL_OK.  Needs no device. */
int zl_token_automaton_check(int vocab, int n_states, const uint32_t* masks, const int32_t* row_ptr, int n_edges,
                             const int32_t* edge_tok, const int32_t* edge_next, const int32_t* default_next, int start);
/* The automaton of `task` from HOST arrays, staged before the call returns; stream-ordered after the steps already
 * enqueued.  masks (n_states, ceil(vocab/32)); row_ptr (n_states + 1) CSR offsets of each state's edges in edge_tok /
 * edge_next (n_edges); default_next (n_states); the task starts in `start`.  n_states = 0 clears the task's automaton (the
 * other arrays are ignored).  Every check runs before anything is enqueued, in this order: a bad task or n_states < 0:
 * ZL_ERR_INVALID_ARG; an automaton under tp_size > 1 without zl_llama_set_vocab_gather: ZL_ERR_UNSUPPORTED (with it,
 * every rank moves the same states from the same rows); constraints not enabled: ZL_ERR_STATE; n_states or n_edges
 * above the caps, an empty mask, a bit at or past vocab, row_ptr not starting at 0, decreasing or not ending at
 * n_edges, edge tokens out of order, repeated or outside their state's mask, or a state out of range:
 * ZL_ERR_INVALID_ARG.  A constrained task makes its batch's pick run the sampler, as a
 * logits processor does, and a beam step over it is refused (ZL_ERR_STATE).  zl_llama_set_sampling leaves it alone. */
int zl_llama_set_constraint(zl_llama_t* m, int task, int n_states, const uint32_t* masks_host, const int32_t* row_ptr_host,
                            int n_edges, const int32_t* edge_tok_host, const int32_t* edge_next_host,
                            const int32_t* default_next_host, int start);
/* The current automaton state of tasks 0 .. B-1 (-1: none) into states_host, once every step enqueued has executed. */
int zl_llama_get_constraint_state(zl_llama_t* m, int32_t* states_host, int B);
/* Copy rows row0 .. row0 + n of task `task`'s layer-`layer` KV cache to the host (the reference's dump_task_buf,
 * rag_buffer_context.h:199-233).  Synchronous.  Plain cache: k_host / v_host get (n, H_kv, d) activation-dtype values and
 * sk_host / sv_host must be NULL.  kv_int8: k_host / v_host get (n, H_kv, d) uint8 codes and sk_host / sv_host (n, H_kv)
 * fp32 scales (either may be NULL to skip it).  H_kv is this rank's kv heads.  Rows past the task's capacity
 * (zl_llama_kv_capacity): ZL_ERR_INVALID_ARG. */
int zl_llama_read_kv(zl_llama_t* m, int layer, int task, int row0, int n, void* k_host, void* v_host, float* sk_host,
                     float* sv_host);
zl_stream_t zl_llama_stream(zl_llama_t* m);
/* bytes the step must read from HBM per rank (weights + lm_head + norms), kernel launches per step. */
int zl_llama_stats(zl_llama_t* m, int B, double* weight_bytes, int* kernels_per_step);
/* Roofline probe for the dominant kernel: enqueue only the W4A16 (or dense) GEMMs of one decode step
 * (every layer's own weights, same PDL chain) `iters` times between CUDA events on the driver's stream.
 * Returns total milliseconds, the number of GEMM launches and their algorithmic bytes. */
int zl_llama_bench_gemms(zl_llama_t* m, int B, int iters, float* ms, int* launches, double* bytes);

/* Prompt prefix cache (enable_prompt_caching of the reference: PrefixCache, src/generator/prefix_cache.hpp:35-117, created
 * at src/generator/batch_generator.cpp:626-645, matched at :1033-1045 and :1120, filled after a prompt's prefill at
 * :1213-1224).  The model owns a device pool of num_blocks blocks of block_tokens KV rows each, for every layer, K and V:
 * pool [layer][K|V][block][block_tokens][H_kv][d] in the cache's element type, and with kv_int8 the fp32 scales
 * [layer][K|V][block][block_tokens][H_kv] beside it, so that codes and scales always move together.  Which blocks hold
 * which tokens is the caller's policy (zhilight_b200/prefix_cache.py keys a block by every block before it).
 * Call after zl_llama_finalize; zl_llama_destroy frees the pool.  block_tokens: 16, 32, 64, 128 or 256, else
 * ZL_ERR_INVALID_ARG; a second call: ZL_ERR_STATE; max_seq * (bytes of one cached row) not a multiple of 16:
 * ZL_ERR_UNSUPPORTED.  A model without a pool allocates nothing for it and runs the same kernels per step. */
int zl_llama_kv_pool_create(zl_llama_t* m, int num_blocks, int block_tokens);
/* Copy n blocks of task `task` into the pool (save: task block task_blocks[i] -> pool block pool_blocks[i]) or out of it
 * (load: pool block pool_blocks[i] -> task block task_blocks[i]).  Task block j is rows [j bt, (j + 1) bt) of the task's
 * buffers.  One kernel launch (k_kv_block_copy) for every layer, K, V and, with kv_int8, the scales.  HOST arrays, staged
 * before the call returns; stream-ordered after every step already enqueued, no device sync.  Loading writes KV rows
 * only: the positions stay with the caller (zl_llama_prefill with pos0 = the loaded length, or a joined segment).
 * Every check runs before anything is enqueued: no pool -> ZL_ERR_STATE; task out of range, a block out of range or past
 * max_seq ((j + 1) bt > max_seq), or a destination block named twice -> ZL_ERR_INVALID_ARG.  A KV arena grants the task
 * the rows the blocks cover first (a save too: it reads them through the task's table); ZL_ERR_KV_FULL when it cannot. */
int zl_llama_kv_blocks_save(zl_llama_t* m, int task, const int32_t* task_blocks, const int32_t* pool_blocks, int n);
int zl_llama_kv_blocks_load(zl_llama_t* m, int task, const int32_t* task_blocks, const int32_t* pool_blocks, int n);
/* Bandwidth probe of the block copy: one warm-up pass, then `iters` passes of the same save (load = 0) or load between
 * CUDA events on the driver's stream, as the k_kv_block_copy launch or (per_range_memcpy != 0) as one cudaMemcpyAsync per
 * (block, layer, tensor) range.  Returns the milliseconds of the timed passes and the bytes one pass reads plus writes.
 * Rewrites the destination blocks; the same checks as zl_llama_kv_blocks_save / load. */
int zl_llama_kv_blocks_bench(zl_llama_t* m, int task, const int32_t* task_blocks, const int32_t* pool_blocks, int n,
                             int load, int per_range_memcpy, int iters, float* ms, double* bytes);

/* Beam search (SearcherImplV1::pick_top_k, src/generator/batch_generator.cpp:1762-1852).  Each beam owns a task slot; the
 * policy that picks beams and slots is the caller's (zhilight_b200/beam_search.py).
 * One beam step: the decode step over tasks 0 .. B-1 (tokens / positions HOST (B) as zl_llama_decode), with the pick
 * replaced by zl_beam_topk on the step's logits -- same CUDA graph, one per (B, G, K, length bucket), no argmax.  groups
 * (G, 2), cum (B) HOST; parent / token / score (G, K) HOST outputs as zl_beam_topk's; logits_host NULL or (B, vocab).
 * Synchronous.  Bad groups, K, cum (NaN or +inf), tokens or positions: ZL_ERR_INVALID_ARG; vocab > 262144, or tp_size > 1 without
 * zl_llama_set_vocab_gather: ZL_ERR_UNSUPPORTED; a task of the batch that samples or has penalties (zl_llama_set_sampling) or logits processors
 * (zl_llama_set_logits_processors) or a constraint (zl_llama_set_constraint): ZL_ERR_STATE; a KV arena that cannot grant
 * the step's rows: ZL_ERR_KV_FULL. */
int zl_llama_beam_step(zl_llama_t* m, const int32_t* tokens, const int32_t* positions, int B, const int32_t* groups, int G,
                       const float* cum, int K, int32_t* parent, int32_t* token, float* score, float* logits_host);
/* Beam forks: one launch copies rows [row0, row1) of task src into task dst for every range ranges_host[i] = {src task,
 * dst task, row0, row1} (HOST (n, 4)), every layer, K and V, and with kv_int8 the fp32 scales.  Staged before the call
 * returns; stream-ordered after the steps already issued, no device sync.  Every check runs before anything is enqueued:
 * a task out of range, rows outside [0, max_seq) or an empty range, a destination named twice, or a task that is both a
 * source and a destination: ZL_ERR_INVALID_ARG.  A KV arena grants every source and destination rows [0, row1) first;
 * ZL_ERR_KV_FULL when it cannot. */
int zl_llama_kv_copy_rows(zl_llama_t* m, const int32_t* ranges_host, int n);

/* Generate until stop on the device (the reference stops a task at eos_id or max_length,
 * src/generator/batch_generator.cpp:1744-1753, 1812-1817).  Each step of zl_llama_generate is the step of
 * zl_llama_step_device -- forward, pick (greedy, or the task's sampling and processors), feedback -- over tasks 0 .. B-1.
 * A running task emits its pick, then stops: 1 when the pick is one of its stop ids, 2 when it has emitted max_new_tokens
 * tokens since its last zl_llama_set_stop, 3 when its next position would reach max_seq.  The emitted token is kept, a
 * stop id included.  A finished task emits nothing until zl_llama_set_stop re-arms it; its row still runs through the
 * forward (the batch shape is baked into the graph) but leaves its KV rows up to its last fed position, its sampler
 * history and its generated-token sequence as they were, and its (token, position) state stays (the emitted token, the
 * position it would be fed).  A task that stopped at position max_seq - 1 re-runs that position while it sits out
 * (there is no later row to write): the same inputs give its last KV row the same values, bit for bit while the batch
 * size and weight format do not couple rows.  Its state position is max_seq, so zl_llama_step_device refuses the batch
 * until zl_llama_set_state moves it.  A task without a stop rule has no stop ids and no budget.
 * Per-task stop rule for zl_llama_generate: up to ZL_MAX_STOP_IDS distinct ids in [0, vocab); max_new_tokens >= 1, or 0
 * for no budget.  Re-arms a finished task and resets its emitted count.  Stream-ordered; host arrays staged before return.
 * Bad task or ids, a repeated id, n_stop > ZL_MAX_STOP_IDS or max_new_tokens < 0: ZL_ERR_INVALID_ARG; tp_size > 1 without
 * zl_llama_set_vocab_gather: ZL_ERR_UNSUPPORTED; a model not finalized: ZL_ERR_STATE. */
#define ZL_MAX_STOP_IDS 8
int zl_llama_set_stop(zl_llama_t* m, int task, const int32_t* stop_ids_host, int n_stop, int max_new_tokens);
/* Up to max_steps (1 .. max_seq) device-resident decode steps of rows 0..B-1, stopping early when all have finished.
 * tokens_host (max_steps, B) step-major: emitted tokens (-1 where a row emitted nothing); n_out_host (B) tokens emitted
 * per task; finish_host (B) 0 running / 1 stop id / 2 max_new_tokens / 3 max_seq; *steps_host steps run.  Synchronous.
 * Starts from the device-resident state (zl_llama_set_state, or earlier steps) and leaves it there, so calls with a small
 * max_steps stream a generation.  The steps run as a CUDA graph per (B, sampling, n-gram launch, attention length
 * bucket): a head kernel and a while-loop conditional node whose body is the decode step plus the stop rules; a call
 * crosses buckets with one graph launch per bucket, without a host sync in between, and syncs once at the end.  A call
 * whose tasks have all finished runs 0 steps and enqueues nothing.  Bad B, max_steps or output pointers:
 * ZL_ERR_INVALID_ARG; tp_size > 1 without zl_llama_set_vocab_gather, or use_graph == 0: ZL_ERR_UNSUPPORTED; a model not finalized: ZL_ERR_STATE.
 * A KV arena first grants each running task min(position + max_steps, max_seq) rows and each finished one the row of its
 * state position: ZL_ERR_KV_FULL when it cannot (retry with a smaller max_steps, or release a task).  Every
 * check runs before anything is enqueued. */
int zl_llama_generate(zl_llama_t* m, int B, int max_steps, int32_t* tokens_host, int32_t* n_out_host,
                      int32_t* finish_host, int* steps_host);

/* KV arena (zl_llama_config_t.kv_rows > 0).  zl_llama_kv_release returns task's rows to the arena (stream order does not
 * matter: no enqueued work is touched, and the rows are zero-filled when granted again); the task's next write is granted
 * fresh rows.  A no-op in the fixed layout.  zl_llama_kv_capacity: the rows the task holds (max_seq in the fixed layout);
 * zl_llama_kv_free_rows: the rows no task holds (0 in the fixed layout).  A bad task: ZL_ERR_INVALID_ARG. */
int zl_llama_kv_release(zl_llama_t* m, int task);
int zl_llama_kv_capacity(zl_llama_t* m, int task, int* rows);
int zl_llama_kv_free_rows(zl_llama_t* m, int* rows);
/* The arena's decisions without a device: replays n_ops operations ops (n_ops, 3) {call, task, rows} on an arena of
 * kv_rows rows (as zl_llama_config_t.kv_rows).  Consecutive operations with the same call id form one call, planned as an
 * entry point plans the rows it writes: rows >= 1 grants the task at least that many rows; rows == 0 releases the task
 * (a call of its own).  Reports results (n_ops) ZL_OK or ZL_ERR_KV_FULL of each operation's call, extents (n_ops,
 * max_batch, 2) {first row, capacity} of every task after it, and the relocation moves (max_moves, 6) {first operation of
 * the call, launch, src row, dst row, rows copied, rows zero-filled} in launch order, *n_moves of them.  Bad arguments, or
 * more than max_moves moves: ZL_ERR_INVALID_ARG. */
int zl_kv_arena_replay(int kv_rows, int max_batch, int max_seq, const int32_t* ops, int n_ops, int32_t* results,
                       int32_t* extents, int32_t* moves, int max_moves, int* n_moves);
/* One k_kv_relocate launch on `stream`: moves (n, 4) {src row, dst row, rows to copy, rows to zero} (DEVICE int32) of the
 * row spaces bases[4 l + t] (DEVICE table; t = 0 K, 1 V, 2 K scales, 3 V scales) of `layers` layers: rows [src, src +
 * copy) to [dst, dst + copy), then rows [dst + copy, dst + copy + zero) zero-filled.  max_rows >= the largest copy + zero;
 * row_bytes % 16 == 0; srow_bytes 0 (no scales) or a multiple of 4.  No move may overlap another's source or
 * destination, and no destination its own source. */
int zl_kv_relocate(void* const* bases, int layers, const int32_t* moves, int n, int max_rows, int row_bytes,
                   int srow_bytes, zl_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* ZHILIGHT_B200_H_ */
