// Kernel parameter block of the W4A16 GEMM variants (host + device).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/zhilight_b200.h"

namespace zl {

// L2 prefetch of the NEXT GEMM's first weight bytes, issued by a v3 kernel as its weight stream drains (a hint: results
// never depend on it).  whole_bytes > 0: the whole range [base, base + whole_bytes).  Otherwise, h > 0: the first h ring
// items of every warp of the successor's v3 launch (grid x subs x warps warps over an n_tiles x G blob of ZLW4I
// records), in the order that warp's producer will request them -- see v3_head_ranges.
struct W4L2Head {
    const uint8_t* base = nullptr;
    int n_tiles = 0, G = 0, grid = 0, subs = 0, warps = 0, h = 0, sub_major = 0;
    unsigned long long whole_bytes = 0;
};

struct W4Params {
    const __half* x;
    int ldx;
    const uint8_t* packed;
    const __half* bias;       // indexed by PACKED row
    const __half* residual;
    __half* y;
    int mc, N, K, epi;
    // fused RMSNorm prologue (ln_w == nullptr: off)
    const __half* ln_w;
    float eps;
    // ZL_EPI_QKV_ROPE
    const float* cos;
    const float* sin;
    __half* q_out;
    const int32_t* token_batch;
    const int32_t* placement;
    __half* const* k_addrs;
    __half* const* v_addrs;
    int num_heads, num_kv_heads, dim_head;
    // weights of the NEXT kernel in the chain: prefetched into L2 as this kernel's weight stream drains (v3 only)
    W4L2Head l2;
    unsigned long long* trace;   // debug: per-CTA globaltimer samples [grid][16] (zl_w4_set_trace)
    int sub_major = 0;   // v3 tile order: sub-CTA s of CTA b starts at tile s * grid + b (else b * SUBS + s)
    int dbg;   // ZL_W4_DEBUG: 1 = skip dequant/MMA (pure weight-stream probe; results are garbage)
    // tensor-parallel exchange inside the GEMM (integer kernel only; comm_dev.cuh).  tp_mode 1 (reduce-in): the
    // activation row is  T(T(sum over ranks of the partial sums pushed by the previous row-parallel GEMM) + x)  -- x is the
    // residual stream -- and CTA 0 stores it to tp_h_out (must not alias x).  tp_mode 2 (push): the epilogue stores the
    // fp16 partial tile into every rank's inbox and the last CTA publishes the epoch flags.
    const void* tp_cd = nullptr;   // const CommDev*
    int tp_mode = 0;
    int tp_index = 0;              // exchange index within the step (< 512): parity of the slot + part of the word tag
    __half* tp_h_out = nullptr;
    // act-order: the staging loop reads x[k_perm[i]] and ln_w[k_perm[i]] (integer kernel only; zl_w4_fused_args_t.k_perm)
    const int32_t* k_perm = nullptr;
    // int8 KV cache (integer kernel, ZL_EPI_QKV_ROPE; zl_w4_fused_args_t.kv_int8): k_addrs / v_addrs point at uint8 code
    // buffers, kv8_sk / kv8_sv at the fp32 scale buffers; kv8_stage (mc, 2, H_kv, d) fp16 scratch, kv8_cnt (mc, 2, H_kv)
    // counters that are 0 on entry and on exit
    int kv8 = 0;
    float* const* kv8_sk = nullptr;
    float* const* kv8_sv = nullptr;
    __half* kv8_stage = nullptr;
    unsigned* kv8_cnt = nullptr;
};

// zl_w4a16_gemm_fused with the L2 head of the successor GEMM as a descriptor (l2 == nullptr: the public whole-range
// prefetch_ptr / prefetch_bytes).  Only the exact-integer kernel issues it, at the tail of its weight stream.
int w4a16_gemm_fused_l2(const zl_w4_fused_args_t* a, const W4L2Head* l2, zl_stream_t stream);
// the variant launch_w4_v3 runs for (mc, N, K, tp_mode) on sm_count SMs; false = none fits
struct V3Plan {
    int nt, warps, subs, stages, rt, pack, grid, smem, sub_major;
};
bool w4_v3_plan(int mc, int N, int K, int tp_mode, int sm_count, V3Plan* plan);

// The kernel that serves M rows of an (N, K) W4 weight, and what it fuses: v3 (exact-integer mma.sync, ZLW4I layout)
// wherever w4_v3_plan finds a variant, else tc (wgmma, ZLW4I layout) where w4_tc_supports, else v2 (fp16 mma.sync, ZLW4
// layout).  None: no W4 kernel takes the shape.  tp_mode and the SM count only choose among v3 variants, never the kernel.
enum class W4Kernel { None, V2, V3, Tc };
struct W4Route {
    W4Kernel kernel = W4Kernel::None;
    int rows = 32;   // rows per launch: up to 256 tokens on the wgmma kernel, 32 on the mma.sync kernels
    V3Plan v3{};     // kernel == V3: the variant launch_w4_v3 runs
    // the wgmma kernel reads x through the TMA engine, so it neither normalises nor gathers it while staging
    bool fuses_rmsnorm() const { return kernel != W4Kernel::Tc; }
    bool gathers_k_perm() const { return kernel == W4Kernel::V3; }
    bool fuses_kv_int8() const { return kernel == W4Kernel::V3; }
    bool exchanges_tp() const { return kernel == W4Kernel::V3; }
};
W4Route w4_route(int M, int N, int K, int tp_mode);

cudaError_t launch_w4_v2(const W4Params& p, bool pdl, cudaStream_t stream);
cudaError_t prepare_w4_v2();
// exact-integer kernel on the ZLW4I layout: the variant w4_route planned for p
cudaError_t launch_w4_v3(const W4Params& p, const V3Plan& plan, bool pdl, cudaStream_t stream);
// descriptor of the L2 head of a successor v3 launch with weights `packed`: its first h ring items per warp, or the
// whole blob when it is at most whole_max bytes; false = the successor does not run the v3 kernel
bool w4_v3_l2_head(const void* packed, int mc, int N, int K, int tp_mode, int sm_count, int h, size_t whole_max,
                   W4L2Head* out);
cudaError_t prepare_w4_v3();
// wgmma / TMA kernel on the ZLW4I layout (w4a16_tc.cu): up to 256 tokens per launch, N % 128 == 0, no fused
// RMSNorm prologue (ln_w is ignored)
cudaError_t launch_w4_tc(const W4Params& p, bool pdl, cudaStream_t stream);
bool w4_tc_supports(int mc, int N, int K);
cudaError_t prepare_w4_tc();
cudaError_t prepare_w8_tc();   // w8_tc.cu

}  // namespace zl
