// wgmma / TMA building blocks shared by the tensor-core kernels (w4a16_tc.cu, w8_tc.cu): bounded mbarrier waits,
// tensor-TMA loads, shared-memory matrix descriptors, wgmma fences, and the host-side tensor-map encoder.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

#include <cuda.h>

namespace zl {

constexpr int kTcRows = 128;   // weight rows per tile: two consumer warpgroups of wgmma M = 64

// ---- PTX wrappers -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// bounded wait: a protocol bug must not hang the GPU (2 s, then the watchdog code is published and the kernel traps)
__device__ __forceinline__ void mbar_wait_wd(uint64_t* bar, uint32_t parity, unsigned* err, unsigned code) {
    if (mbar_try_wait(bar, parity)) return;
    // the spin itself touches nothing but the barrier (a %globaltimer read per poll costs hundreds of cycles of wake-up
    // latency on every hand-over); the SM clock is sampled once per 2048 polls
    const long long t0 = clock64();
    unsigned spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 2047u) == 0 && clock64() - t0 > 4000000000ll) {
            if (err) atomicExch(err, code);
            __threadfence_system();
            __trap();
        }
    }
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::
            "r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_load_3d_hint(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar,
                                                 uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, "
        "%4}], [%5], %6;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d_hint(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                                 uint64_t* bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, "
        "%4, %5}], [%6], %7;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
// tagged 8-byte words of the partial-tile exchange: {payload, tag}, one atomic store / load each
__device__ __forceinline__ void tc_st_tag(uint2* p, uint32_t data, uint32_t tag) {
    asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(data), "r"(tag) : "memory");
}
__device__ __forceinline__ uint2 tc_ld_tag(const uint2* p) {
    uint2 v;
    asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}
// K-major, 128-byte-swizzled shared-memory matrix descriptor of wgmma: start address >> 4, LBO (unused for swizzled K-major,
// canonical value 1), SBO = 1024 B between 8-row groups, layout type 1 (SWIZZLE_128B).  The tile must be 1024-byte aligned;
// +2 on the descriptor advances K by 32 bytes inside the swizzle atom.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t saddr) {
    uint64_t d = (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// named barrier of the two consumer warpgroups (the producer warp does not take part)
__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ---- host: cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn tc_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

// 2-D row-major tensor (rows, cols) of `elem_bytes`-byte elements, row pitch ld_bytes; box = 128 bytes of a row x box_rows
// rows, 128-byte swizzle (the K-major wgmma operand layout), out-of-bounds rows / columns read as zero
inline bool tc_make_map_2d(CUtensorMap* map, const void* base, CUtensorMapDataType dt, int elem_bytes, uint64_t rows,
                           uint64_t cols, uint64_t ld_bytes, uint32_t box_rows) {
    EncodeTiledFn enc = tc_encode_fn();
    if (!enc) return false;
    const cuuint64_t gdim[2] = {cols, rows};
    const cuuint64_t gstride[1] = {ld_bytes};
    const cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), box_rows};
    const cuuint32_t estr[2] = {1u, 1u};
    return enc(map, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// general tiled map: rank <= 5, dims / box fastest-first, strides (bytes) of dims 1 .. rank-1
inline bool tc_make_map_nd(CUtensorMap* map, const void* base, CUtensorMapDataType dt, int rank, const uint64_t* dims,
                           const uint64_t* strides, const uint32_t* box, CUtensorMapSwizzle swz) {
    EncodeTiledFn enc = tc_encode_fn();
    if (!enc || rank < 1 || rank > 5) return false;
    cuuint64_t gdim[5], gstride[4];
    cuuint32_t b[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        b[i] = box[i];
        estr[i] = 1u;
        if (i > 0) gstride[i - 1] = strides[i - 1];
    }
    return enc(map, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstride, b, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// per-device scratch of the split-k reductions: fp32 / int32 partial tiles, arrival counters, watchdog word
struct TcDeviceState {
    float* ws = nullptr;
    uint2* ws_ll = nullptr;            // W4 kernel: tagged partial-tile words {fp32 bits, tag}, all zero between launches
    size_t ws_ll_bytes = 0;
    unsigned* counters = nullptr;
    unsigned* err = nullptr;
    size_t ws_bytes = 0;
};
constexpr size_t kTcWsLlBytes = 80ull << 20;   // >= 2 slots x 132 CTAs x 256 tokens x 128 rows x 8 B
constexpr size_t kTcWsBytes = 64ull << 20;   // >= 2 x 132 items x 256 tokens x 128 rows x 4 B
constexpr int kTcMaxTiles = 8192;
TcDeviceState* tc_state();                   // w4a16_tc.cu; nullptr before prepare_w4_tc() ran on the current device

}  // namespace zl
