// Shared device helpers for the sm_90a kernels (mbarrier, bulk-TMA, PDL, mma.sync, packing).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "../../include/zhilight_b200.h"

#define ZL_CHECK_ARG(cond)                                                             \
    do {                                                                               \
        if (!(cond)) {                                                                 \
            zl_set_last_error(__FILE__, __LINE__, "invalid argument: " #cond);         \
            return ZL_ERR_INVALID_ARG;                                                 \
        }                                                                              \
    } while (0)

#define ZL_CHECK_SUPPORTED(cond)                                                       \
    do {                                                                               \
        if (!(cond)) {                                                                 \
            zl_set_last_error(__FILE__, __LINE__, "unsupported: " #cond);              \
            return ZL_ERR_UNSUPPORTED;                                                 \
        }                                                                              \
    } while (0)

#define ZL_CHECK_CUDA(expr)                                                            \
    do {                                                                               \
        cudaError_t _e = (expr);                                                       \
        if (_e != cudaSuccess) {                                                       \
            zl_set_last_error(__FILE__, __LINE__, cudaGetErrorString(_e));             \
            return ZL_ERR_CUDA;                                                        \
        }                                                                              \
    } while (0)

#define ZL_CHECK_LAUNCH() ZL_CHECK_CUDA(cudaGetLastError())

extern "C" void zl_set_last_error(const char* file, int line, const char* msg);
extern "C" void zl_count_launch(void);

namespace zl {

constexpr int kWarp = 32;

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// zl_prepare() on the CURRENT device unless it already ran there (w4a16_api.cu).  Called lazily before the first launch
// that needs it: opt-in shared memory must be set outside of stream capture.
int prepare_once();

// SM count of the CURRENT device, cached per device id (one process may drive several devices: one host thread per
// GPU in the reference engine, engine.cpp:115-117).  A benign race only repeats the query.
inline int device_sm_count() {
    static int cache[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && cache[dev] > 0) return cache[dev];
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
    if (dev >= 0 && dev < 64) cache[dev] = n;
    return n;
}

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  Every kernel in the decode chain calls pdl_trigger() as
// early as possible (its dependents only prefetch read-only weights before their own pdl_wait())
// and pdl_wait() before touching anything a predecessor produced.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_trigger() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

// Launch helper: sets the PDL attribute when `pdl` is non-zero.
template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                          cudaStream_t stream, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    zl_count_launch();
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---------------------------------------------------------------------------------------------
// mbarrier + bulk (non-tensor) TMA copies global -> shared::cta
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    // make mbarrier.init visible to the async (TMA) proxy
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// 1-D bulk copy (TMA engine, SASS UBLKCP): bytes % 16 == 0, src/dst 16-B aligned.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// same copy, tagged evict-first in L2: a weight stream is read exactly once per step and must not push the
// prefetched weights of the NEXT kernel (l2_prefetch below) out of the 50 MB L2
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar,
                                              uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
// fire-and-forget prefetch of [p, p+bytes) into L2 (bytes % 16 == 0, p 16-B aligned)
__device__ __forceinline__ void l2_prefetch(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
// each (cta, warp) of the grid prefetches its strided share of [base, base+bytes) in 4 KB pieces; call from lane 0
__device__ __forceinline__ void l2_prefetch_share(const uint8_t* base, size_t bytes, int part, int parts) {
    constexpr size_t kChunk = 4096;
    const size_t n_chunks = (bytes + kChunk - 1) / kChunk;
    for (size_t c = (size_t)part; c < n_chunks; c += (size_t)parts) {
        const size_t off = c * kChunk;
        const size_t len = bytes - off < kChunk ? bytes - off : kChunk;
        l2_prefetch(base + off, (uint32_t)(len & ~(size_t)15));
    }
}

// ---------------------------------------------------------------------------------------------
// loads
// ---------------------------------------------------------------------------------------------
// L2-only (bypass L1): used for activations produced by a predecessor kernel under PDL.
__device__ __forceinline__ uint4 ld_cg_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ld_cg_u2(const void* p) {
    uint2 r;
    asm volatile("ld.global.cg.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
// streaming read-only data (weights, KV): no L1 allocation
__device__ __forceinline__ uint4 ld_nc_na_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// ---------------------------------------------------------------------------------------------
// warp-level tensor-core MMA (the wgmma kernels live in w4a16_tc.cu and w8_tc.cu)
// D(16x8,f32) += A(16x16,f16,row) * B(16x8,f16,col)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_16816_f16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1,
                                              const float (&c)[4]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
        "{%10,%11,%12,%13};"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(c[0]), "f"(c[1]), "f"(c[2]),
          "f"(c[3]));
}
__device__ __forceinline__ void mma_16816_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1,
                                               const float (&c)[4]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
        "{%10,%11,%12,%13};"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(c[0]), "f"(c[1]), "f"(c[2]),
          "f"(c[3]));
}

template <uint32_t A, uint32_t B>
__device__ __forceinline__ uint32_t lop3_and_or(uint32_t x) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xea;" : "=r"(r) : "r"(x), "n"(A), "n"(B));   // (x & A) | B
    return r;
}

// ---------------------------------------------------------------------------------------------
// dtype helpers: T in {__half, __nv_bfloat16}
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }

template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }

template <typename T>
__device__ __forceinline__ float round_to(float v) { return to_f32<T>(from_f32<T>(v)); }

// unpack 8 x 16-bit values held in a uint4 into floats
template <typename T>
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    const T* p = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = to_f32<T>(p[i]);
}
template <typename T>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    uint4 u;
    T* p = reinterpret_cast<T*>(&u);
#pragma unroll
    for (int i = 0; i < 8; ++i) p[i] = from_f32<T>(f[i]);
    return u;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }   // activation.cuh:12-14
__device__ __forceinline__ float gelu_f(float x) {                                    // activation.cuh:8-10
    return 0.5f * x * (1.0f + tanhf(0.7978845608028654f * x * (1.0f + 0.044715f * x * x)));
}

}  // namespace zl
