// Tensor-parallel exchange over NVLink peer memory: one-shot all-reduce (fp16/bf16 or int8 group-32 payload)
// fused with the residual add, and a small one-shot all-gather.  One process per GPU; the symmetric buffers are
// cudaMalloc'ed per rank and mapped into the peers with CUDA IPC (handles travel over torch.distributed).
//
// Replaces ModelContext::reduce_sum / reduce_sum2 / reduce_tp_int8 (reference src/model/model_context.cpp:203-326:
// ncclAllReduce, or quant -> grouped Send/Recv -> dequant-sum-requant -> grouped Send/Recv -> dequant = two NCCL
// groups + 3-4 kernels) and the residual add that follows it (src/nn/block/block.cpp:124-125, block_kernel.cu:7-50)
// with ONE kernel: every rank stores its partial sum straight into each peer's inbox, publishes a flag, waits for
// the peers' flags and reduces in rank order (deterministic).  Decode messages are <= 512 KiB, so latency, not
// bandwidth, is the bound: one NVLink store round trip instead of two collectives.
//
// The stand-alone group-32 int8 kernels of the reference (src/nn/quant/int8/quant_reduce_kernel.cu:14-38, 105-140,
// 201-274) are provided bit-exactly at the end of this file.
#include "common.cuh"
#include "comm_dev.cuh"

#include <cstring>
#include <vector>

namespace zl {

constexpr int kCommThreads = 256;

// One-shot all-reduce of `n` elements (n % 8 == 0 for 16-bit payload; n % 32 == 0 for int8 payload).
//   out = T( T(sum_r partial_r) + residual )   (residual may be null; out may alias residual)
// int8 != 0: every contribution is quantised to int8 with one T scale per 32 values (the reference's
// quant_group_32 format) and all ranks sum the same ws quantised vectors in rank order.
template <typename T>
__global__ void __launch_bounds__(kCommThreads)
k_allreduce_one_shot(const CommDev* __restrict__ cd, const T* __restrict__ partial, const T* __restrict__ residual,
                     T* __restrict__ out, int n, int int8) {
    __shared__ unsigned long long s_epoch;
    const CommDev c = *cd;
    pdl_trigger();
    pdl_wait();
    if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile unsigned long long*>(c.epoch);
    __syncthreads();
    const unsigned long long e = s_epoch;
    const int parity = (int)(e & 1ull);
    const int n_cta = gridDim.x;
    // this CTA's contiguous chunk, multiple of 32 elements
    const int groups = n / 32;
    const int g0 = (int)((long long)groups * blockIdx.x / n_cta), g1 = (int)((long long)groups * (blockIdx.x + 1) / n_cta);
    const int e0 = g0 * 32, e1 = g1 * 32;
    const size_t my_slot = ((size_t)parity * c.ws + c.rank) * c.slot_bytes;

    // ---- push my chunk into every peer's inbox ----
    if (!int8) {
        for (int i = e0 + threadIdx.x * 8; i < e1; i += kCommThreads * 8) {
            const uint4 v = ld_cg_u4(partial + i);
            for (int r = 0; r < c.ws; ++r)
                if (r != c.rank) *reinterpret_cast<uint4*>(c.inbox[r] + my_slot + (size_t)i * sizeof(T)) = v;
        }
    } else {
        // payload: [n] int8 then [n/32] T scales ; one warp per 32-group
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (int gidx = g0 + warp; gidx < g1; gidx += kCommThreads / 32) {
            const float v = to_f32<T>(__ldcg(partial + gidx * 32 + lane));
            float amax = fabsf(v);
            amax = round_to<T>(warp_max(amax));   // warpReduceMaxB<T>: the maximum is carried in T
            const int8_t q = (int8_t)nearbyintf(v * 127.0f / amax);
            const T sc = from_f32<T>(amax / 127.0f);
            // the own slot is written too: every rank then sums the SAME ws quantised contributions in rank
            // order, so all ranks hold bit-identical results (the reference gets that from its all-gather)
            for (int r = 0; r < c.ws; ++r) {
                uint8_t* base = c.inbox[r] + my_slot;
                reinterpret_cast<int8_t*>(base)[gidx * 32 + lane] = q;
                if (lane == 0) reinterpret_cast<T*>(base + n)[gidx] = sc;
            }
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < c.ws && (int)threadIdx.x != c.rank) {
        unsigned long long* flag = reinterpret_cast<unsigned long long*>(c.inbox[threadIdx.x] +
                                                                        comm_flags_offset(c.ws, c.slot_bytes)) +
                                   (size_t)c.rank * kCommMaxCtas + blockIdx.x;
        st_release_sys(flag, e + 1);
    }
    // ---- wait for the same chunk of every peer ----
    if (threadIdx.x < c.ws && (int)threadIdx.x != c.rank) {
        const unsigned long long* flag = reinterpret_cast<const unsigned long long*>(
                                             c.inbox[c.rank] + comm_flags_offset(c.ws, c.slot_bytes)) +
                                         (size_t)threadIdx.x * kCommMaxCtas + blockIdx.x;
        while (ld_acquire_sys(flag) < e + 1) {
        }
    }
    __syncthreads();

    // ---- reduce in rank order + residual ----
    const uint8_t* mine = c.inbox[c.rank];
    for (int i = e0 + threadIdx.x * 8; i < e1; i += kCommThreads * 8) {
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        if (!int8) {
            for (int r = 0; r < c.ws; ++r) {
                uint4 v = (r == c.rank) ? ld_cg_u4(partial + i)
                                        : ld_cg_u4(mine + ((size_t)parity * c.ws + r) * c.slot_bytes + (size_t)i * sizeof(T));
                float f[8];
                unpack8<T>(v, f);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] += f[k];
            }
        } else {
            for (int r = 0; r < c.ws; ++r) {
                const uint8_t* base = mine + ((size_t)parity * c.ws + r) * c.slot_bytes;
                const uint2 qv = ld_cg_u2(base + i);
                const float sc = to_f32<T>(__ldcg(reinterpret_cast<const T*>(base + n) + i / 32));
                const int8_t* q = reinterpret_cast<const int8_t*>(&qv);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] += (float)q[k] * sc;
            }
        }
        if (residual) {
            float rf[8];
            unpack8<T>(ld_cg_u4(residual + i), rf);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] = round_to<T>(acc[k]) + rf[k];   // T(sum) then the T add of block_kernel.cu
        }
        *reinterpret_cast<uint4*>(out + i) = pack8<T>(acc);
    }
    // ---- last CTA out advances the epoch ----
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(c.done, 1u) == (unsigned)n_cta - 1) {
            *c.done = 0;
            __threadfence();
            *reinterpret_cast<volatile unsigned long long*>(c.epoch) = e + 1;
        }
    }
}

// one-shot all-gather of `bytes` (multiple of 16, <= slot_bytes) per rank: out[r] = in of rank r
__global__ void __launch_bounds__(kCommThreads)
k_allgather_small(const CommDev* __restrict__ cd, const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int bytes) {
    __shared__ unsigned long long s_epoch;
    const CommDev c = *cd;
    pdl_trigger();
    pdl_wait();
    if (threadIdx.x == 0) s_epoch = *reinterpret_cast<volatile unsigned long long*>(c.epoch);
    __syncthreads();
    const unsigned long long e = s_epoch;
    const int parity = (int)(e & 1ull);
    const size_t my_slot = ((size_t)parity * c.ws + c.rank) * c.slot_bytes;
    for (int i = threadIdx.x * 16; i < bytes; i += kCommThreads * 16) {
        const uint4 v = ld_cg_u4(in + i);
        for (int r = 0; r < c.ws; ++r)
            if (r != c.rank) *reinterpret_cast<uint4*>(c.inbox[r] + my_slot + i) = v;
        *reinterpret_cast<uint4*>(out + (size_t)c.rank * bytes + i) = v;
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < c.ws && (int)threadIdx.x != c.rank) {
        unsigned long long* flag = reinterpret_cast<unsigned long long*>(c.inbox[threadIdx.x] +
                                                                        comm_flags_offset(c.ws, c.slot_bytes)) +
                                   (size_t)c.rank * kCommMaxCtas;
        st_release_sys(flag, e + 1);
        const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(
                                             c.inbox[c.rank] + comm_flags_offset(c.ws, c.slot_bytes)) +
                                         (size_t)threadIdx.x * kCommMaxCtas;
        while (ld_acquire_sys(mine) < e + 1) {
        }
    }
    __syncthreads();
    const uint8_t* base = c.inbox[c.rank];
    for (int r = 0; r < c.ws; ++r) {
        if (r == c.rank) continue;
        for (int i = threadIdx.x * 16; i < bytes; i += kCommThreads * 16)
            *reinterpret_cast<uint4*>(out + (size_t)r * bytes + i) =
                ld_cg_u4(base + ((size_t)parity * c.ws + r) * c.slot_bytes + i);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        *reinterpret_cast<volatile unsigned long long*>(c.epoch) = e + 1;
    }
}

// ---- the reference's stand-alone group-32 kernels (bit-exact restatements) ----
// quant_group_32 (quant_reduce_kernel.cu:14-38): one warp per group
template <typename T>
__global__ void k_quant_group_32(const T* __restrict__ in, int8_t* __restrict__ out, T* __restrict__ scale, size_t M) {
    const size_t m = (size_t)blockIdx.x * blockDim.y + threadIdx.y;
    if (m >= M) return;
    const float v = to_f32<T>(in[m * 32 + threadIdx.x]);
    const float amax = round_to<T>(warp_max(fabsf(v)));
    out[m * 32 + threadIdx.x] = (int8_t)nearbyintf(v * 127.0f / amax);
    if (threadIdx.x == 0) scale[m] = from_f32<T>(amax / 127.0f);
}
// dequant_sum_quant_g32 (quant_reduce_kernel.cu:243-274)
template <typename T>
__global__ void k_dequant_sum_quant_g32(const T* __restrict__ my, const int8_t* __restrict__ q_others,
                                        const T* __restrict__ s_others, int8_t* __restrict__ out_q,
                                        T* __restrict__ out_s, size_t M, int ws) {
    const size_t m = (size_t)blockIdx.x * blockDim.y + threadIdx.y;
    if (m >= M) return;
    const size_t off = m * 32 + threadIdx.x;
    float sum = to_f32<T>(my[off]);
    for (int r = 0; r < ws - 1; ++r)
        sum += (float)q_others[off + (size_t)r * M * 32] * to_f32<T>(s_others[(size_t)r * M + m]);
    const float amax = round_to<T>(warp_max(fabsf(sum)));
    out_q[off] = (int8_t)nearbyintf(sum * 127.0f / amax);
    if (threadIdx.x == 0) out_s[m] = from_f32<T>(amax / 127.0f);
}
// dequant_group_32 / dequant_group_fuse_add (quant_reduce_kernel.cu:105-140, 201-240)
template <typename T>
__global__ void k_dequant_group_32(const int8_t* __restrict__ q, const T* __restrict__ scale, const T* __restrict__ add,
                                   T* __restrict__ out, size_t M) {
    const size_t m = (size_t)blockIdx.x * blockDim.y + threadIdx.y;
    if (m >= M) return;
    const size_t off = m * 32 + threadIdx.x;
    float v = (float)q[off] * to_f32<T>(scale[m]);
    if (add) v += to_f32<T>(add[off]);
    out[off] = from_f32<T>(v);
}

}  // namespace zl

using namespace zl;

struct zl_comm {
    int rank = 0, ws = 1;
    size_t slot_bytes = 0;
    uint8_t* local = nullptr;                  // this rank's symmetric buffer
    uint8_t* peers[kCommMaxRanks] = {};        // mapped peer buffers (peers[rank] == local)
    CommDev* dev = nullptr;
    unsigned long long* epoch = nullptr;
    unsigned int* done = nullptr;
    unsigned int* ll_step = nullptr;
    bool opened = false;
};

extern "C" int zl_comm_create(int rank, int world_size, size_t max_elems_16bit, zl_comm_t** out) {
    ZL_CHECK_ARG(out && world_size >= 1 && world_size <= kCommMaxRanks && rank >= 0 && rank < world_size);
    ZL_CHECK_ARG(max_elems_16bit > 0 && max_elems_16bit % 32 == 0);
    zl_comm* c = new zl_comm();
    c->rank = rank;
    c->ws = world_size;
    c->slot_bytes = (max_elems_16bit * 2 + 127) & ~(size_t)127;
    const size_t total = comm_total_bytes(world_size, c->slot_bytes);
    ZL_CHECK_CUDA(cudaMalloc((void**)&c->local, total));
    ZL_CHECK_CUDA(cudaMemset(c->local, 0, total));
    ZL_CHECK_CUDA(cudaMalloc((void**)&c->dev, sizeof(CommDev)));
    ZL_CHECK_CUDA(cudaMalloc((void**)&c->epoch, 8));
    ZL_CHECK_CUDA(cudaMalloc((void**)&c->done, 4));
    ZL_CHECK_CUDA(cudaMemset(c->epoch, 0, 8));
    ZL_CHECK_CUDA(cudaMemset(c->done, 0, 4));
    ZL_CHECK_CUDA(cudaMalloc((void**)&c->ll_step, 4));
    ZL_CHECK_CUDA(cudaMemset(c->ll_step, 0, 4));
    c->peers[rank] = c->local;
    if (world_size == 1) {
        CommDev h = {};
        h.inbox[0] = c->local;
        h.rank = 0;
        h.ws = 1;
        h.slot_bytes = c->slot_bytes;
        h.epoch = c->epoch;
        h.done = c->done;
        h.ll_step = c->ll_step;
        ZL_CHECK_CUDA(cudaMemcpy(c->dev, &h, sizeof(h), cudaMemcpyHostToDevice));
        c->opened = true;
    }
    ZL_CHECK_CUDA(cudaDeviceSynchronize());
    *out = c;
    return ZL_OK;
}

extern "C" int zl_comm_ipc_handle_bytes(void) { return (int)sizeof(cudaIpcMemHandle_t); }

extern "C" int zl_comm_get_ipc_handle(zl_comm_t* c, void* handle_out) {
    ZL_CHECK_ARG(c && handle_out);
    cudaIpcMemHandle_t h;
    ZL_CHECK_CUDA(cudaIpcGetMemHandle(&h, c->local));
    memcpy(handle_out, &h, sizeof(h));
    return ZL_OK;
}

// handles_all: world_size consecutive cudaIpcMemHandle_t, index = rank (the own entry is ignored)
extern "C" int zl_comm_open_peers(zl_comm_t* c, const void* handles_all) {
    ZL_CHECK_ARG(c && handles_all);
    if (c->opened) return ZL_OK;
    const cudaIpcMemHandle_t* hs = static_cast<const cudaIpcMemHandle_t*>(handles_all);
    for (int r = 0; r < c->ws; ++r) {
        if (r == c->rank) continue;
        void* p = nullptr;
        ZL_CHECK_CUDA(cudaIpcOpenMemHandle(&p, hs[r], cudaIpcMemLazyEnablePeerAccess));
        c->peers[r] = static_cast<uint8_t*>(p);
    }
    CommDev h = {};
    for (int r = 0; r < c->ws; ++r) h.inbox[r] = c->peers[r];
    h.rank = c->rank;
    h.ws = c->ws;
    h.slot_bytes = c->slot_bytes;
    h.epoch = c->epoch;
    h.done = c->done;
    h.ll_step = c->ll_step;
    ZL_CHECK_CUDA(cudaMemcpy(c->dev, &h, sizeof(h), cudaMemcpyHostToDevice));
    c->opened = true;
    return ZL_OK;
}

extern "C" void zl_comm_destroy(zl_comm_t* c) {
    if (!c) return;
    cudaDeviceSynchronize();
    for (int r = 0; r < c->ws; ++r)
        if (r != c->rank && c->peers[r]) cudaIpcCloseMemHandle(c->peers[r]);
    cudaFree(c->local);
    cudaFree(c->dev);
    cudaFree(c->epoch);
    cudaFree(c->done);
    cudaFree(c->ll_step);
    delete c;
}

extern "C" int zl_comm_rank(zl_comm_t* c) { return c ? c->rank : -1; }
extern "C" const void* zl_comm_device_state(zl_comm_t* c) { return (c && c->opened) ? c->dev : nullptr; }
extern "C" size_t zl_comm_slot_bytes(zl_comm_t* c) { return c ? c->slot_bytes : 0; }

__global__ void k_comm_ll_step(unsigned int* step) {
    pdl_trigger();
    pdl_wait();
    if (threadIdx.x == 0) *step += 1u;
}
// once per decode step that uses the tagged exchange, before its first GEMM: every rank runs the same steps, so the counters
// (and with them the tags) agree without any communication
extern "C" int zl_comm_ll_begin_step(zl_comm_t* c, zl_stream_t stream) {
    ZL_CHECK_ARG(c && c->opened);
    ZL_CHECK_CUDA(launch(k_comm_ll_step, dim3(1), dim3(32), 0, stream, false, c->ll_step));
    return ZL_OK;
}
extern "C" int zl_comm_world_size(zl_comm_t* c) { return c ? c->ws : -1; }
extern "C" int zl_comm_local_buffer(zl_comm_t* c, void** base, size_t* bytes) {
    ZL_CHECK_ARG(c && base && bytes);
    *base = c->local;
    *bytes = comm_total_bytes(c->ws, c->slot_bytes);
    return ZL_OK;
}

extern "C" int zl_allreduce_one_shot(zl_comm_t* c, const void* partial, const void* residual, void* out, size_t n,
                                     int dtype, int int8_payload, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(c && partial && out && n > 0 && n % 32 == 0);
    if (!c->opened) {
        zl_set_last_error(__FILE__, __LINE__, "zl_comm: peers not opened");
        return ZL_ERR_STATE;
    }
    ZL_CHECK_ARG(n * 2 <= c->slot_bytes && n < (size_t)1 << 30);
    ZL_CHECK_SUPPORTED(dtype == ZL_F16 || dtype == ZL_BF16);
    int ctas = (int)(n / 2048);   // >= 2048 elements per CTA
    if (ctas < 1) ctas = 1;
    if (ctas > kCommMaxCtas) ctas = kCommMaxCtas;
    if (dtype == ZL_F16)
        ZL_CHECK_CUDA(launch(k_allreduce_one_shot<__half>, dim3(ctas), dim3(kCommThreads), 0, stream, pdl != 0,
                             (const CommDev*)c->dev, (const __half*)partial, (const __half*)residual, (__half*)out,
                             (int)n, int8_payload));
    else
        ZL_CHECK_CUDA(launch(k_allreduce_one_shot<__nv_bfloat16>, dim3(ctas), dim3(kCommThreads), 0, stream, pdl != 0,
                             (const CommDev*)c->dev, (const __nv_bfloat16*)partial, (const __nv_bfloat16*)residual,
                             (__nv_bfloat16*)out, (int)n, int8_payload));
    return ZL_OK;
}

extern "C" int zl_allgather_small(zl_comm_t* c, const void* in, void* out, size_t bytes, int pdl, zl_stream_t stream) {
    ZL_CHECK_ARG(c && in && out && bytes > 0 && bytes % 16 == 0);
    if (!c->opened) {
        zl_set_last_error(__FILE__, __LINE__, "zl_comm: peers not opened");
        return ZL_ERR_STATE;
    }
    ZL_CHECK_ARG(bytes <= c->slot_bytes);
    ZL_CHECK_CUDA(launch(k_allgather_small, dim3(1), dim3(kCommThreads), 0, stream, pdl != 0, (const CommDev*)c->dev,
                         (const uint8_t*)in, (uint8_t*)out, (int)bytes));
    return ZL_OK;
}

#define ZL_DISPATCH_T16(dtype, ...)                        \
    if ((dtype) == ZL_F16) {                               \
        using scalar_t = __half;                           \
        __VA_ARGS__                                        \
    } else if ((dtype) == ZL_BF16) {                       \
        using scalar_t = __nv_bfloat16;                    \
        __VA_ARGS__                                        \
    } else {                                               \
        ZL_CHECK_SUPPORTED((dtype) == ZL_F16 || (dtype) == ZL_BF16); \
    }

extern "C" int zl_quant_group_32(const void* in, int8_t* out_q, void* out_scale, size_t M, int dtype,
                                 zl_stream_t stream) {
    ZL_CHECK_ARG(in && out_q && out_scale && M > 0);
    dim3 block(32, 8), grid((unsigned)((M + 7) / 8));
    ZL_DISPATCH_T16(dtype, { k_quant_group_32<scalar_t><<<grid, block, 0, stream>>>((const scalar_t*)in, out_q, (scalar_t*)out_scale, M); })
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_dequant_sum_quant_g32(const void* my, const int8_t* q_others, const void* scale_others,
                                        int8_t* out_q, void* out_scale, size_t M, int world_size, int dtype,
                                        zl_stream_t stream) {
    ZL_CHECK_ARG(my && q_others && scale_others && out_q && out_scale && M > 0);
    ZL_CHECK_ARG(world_size == 2 || world_size == 4 || world_size == 8);   // quant_reduce_kernel.cu:290
    dim3 block(32, 8), grid((unsigned)((M + 7) / 8));
    ZL_DISPATCH_T16(dtype, {
        k_dequant_sum_quant_g32<scalar_t><<<grid, block, 0, stream>>>((const scalar_t*)my, q_others,
                                                                      (const scalar_t*)scale_others, out_q,
                                                                      (scalar_t*)out_scale, M, world_size);
    })
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_dequant_group_32(const int8_t* q, const void* scale, const void* add, void* out, size_t M, int dtype,
                                   zl_stream_t stream) {
    ZL_CHECK_ARG(q && scale && out && M > 0);
    dim3 block(32, 8), grid((unsigned)((M + 7) / 8));
    ZL_DISPATCH_T16(dtype, {
        k_dequant_group_32<scalar_t><<<grid, block, 0, stream>>>(q, (const scalar_t*)scale, (const scalar_t*)add,
                                                                 (scalar_t*)out, M);
    })
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}
