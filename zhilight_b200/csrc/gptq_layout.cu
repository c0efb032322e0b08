// Load-time integer layout transforms (bit-exact with the reference) and the ZLW4 tile packer.
//
// Reference behaviour restated (not copied): src/nn/quant/gptq/qdq_4.cuh:16-35 (nibble shuffle),
// q_gemm.cu:794-872 (act-order gather + shuffle), utils.cu:25-58 (AWQ zero de-interleave),
// utils.cu:61-118 (zero +1 / subtract 8), utils.cu:121-174 (AWQ -> GPTQ packing),
// utils.cu:177-214 (q4 -> q8), q_gemm_k_major.cu:843-905 (dequant to fp16).
#include "common.cuh"
#include "w4_layout.cuh"

namespace zl {

// ---- nibble shuffle: [q0..q7] -> low16 = [q0,q2,q4,q6], high16 = [q1,q3,q5,q7] ----------------
__device__ __forceinline__ uint32_t shuffle_word(uint32_t w) {
    uint32_t out = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        out |= ((w >> (8 * i)) & 0xFu) << (4 * i);
        out |= ((w >> (8 * i + 4)) & 0xFu) << (4 * i + 16);
    }
    return out;
}

__global__ void k_shuffle_words(uint32_t* __restrict__ w, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) w[i] = shuffle_word(w[i]);
}

// act-order gather: new nibble row r (of the K x N nibble matrix) = old row q_perm[r]
__global__ void k_make_sequential(const uint32_t* __restrict__ w, uint32_t* __restrict__ out,
                                  const int32_t* __restrict__ q_perm, int K8, int N) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    int r8 = blockIdx.y;
    if (n >= N) return;
    uint32_t dst = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int src_row = q_perm[r8 * 8 + i];
        uint32_t v = (w[(size_t)(src_row >> 3) * N + n] >> ((src_row & 7) * 4)) & 0xFu;
        dst |= v << (4 * i);
    }
    out[(size_t)r8 * N + n] = dst;
}

__global__ void k_inc_zero(uint32_t* __restrict__ w, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t q = w[i];
    // per-nibble (z + 1) & 15 without carries between nibbles
    uint32_t lo = (q & 0x77777777u) + 0x11111111u;          // add 1 to low 3 bits of each nibble
    uint32_t r = lo ^ (q & 0x88888888u);                     // fold the top bit back in (xor == add mod 16)
    w[i] = r;
}

__global__ void k_sub8(uint32_t* __restrict__ w, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) w[i] ^= 0x88888888u;   // (q>=8 ? q-8 : q+8) == q ^ 8 per nibble
}

__global__ void k_q4_to_q8(const uint32_t* __restrict__ in, uint2* __restrict__ out, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t q = in[i];
    uint2 o;
    o.x = (q & 0xFu) | ((q & 0xF0u) << 4) | ((q & 0xF00u) << 8) | ((q & 0xF000u) << 12);
    q >>= 16;
    o.y = (q & 0xFu) | ((q & 0xF0u) << 4) | ((q & 0xF00u) << 8) | ((q & 0xF000u) << 12);
    out[i] = o;
}

__device__ __forceinline__ uint32_t awq_deinterleave(uint32_t q) {
    // out nibble s = in nibble {0,4,1,5,2,6,3,7}[s]
    uint32_t o = 0;
    const int de[8] = {0, 4, 1, 5, 2, 6, 3, 7};
#pragma unroll
    for (int s = 0; s < 8; ++s) o |= ((q >> (de[s] * 4)) & 0xFu) << (s * 4);
    return o;
}

__global__ void k_awq_un_shuffle(uint32_t* __restrict__ w, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) w[i] = awq_deinterleave(w[i]);
}

// AWQ (K, N/8) -> GPTQ (K/8, N); one thread per (k8, n8) 8x8 nibble block
__global__ void k_awq_shuffle(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int K8, int N8,
                              int use_exllama) {
    int n8 = blockIdx.x * blockDim.x + threadIdx.x;
    int k8 = blockIdx.y;
    if (n8 >= N8) return;
    uint32_t rows[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) rows[r] = awq_deinterleave(in[(size_t)(k8 * 8 + r) * N8 + n8]);
    const int sfl[8] = {0, 2, 4, 6, 1, 3, 5, 7};
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        uint32_t q = 0;
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            int r = use_exllama ? sfl[s] : s;
            q |= ((rows[r] >> (4 * c)) & 0xFu) << (4 * s);
        }
        out[(size_t)k8 * (N8 * 8) + n8 * 8 + c] = q;
    }
}

template <typename T>
__global__ void k_transpose(const T* __restrict__ in, T* __restrict__ out, int rows, int cols) {
    __shared__ T tile[32][33];
    int c = blockIdx.x * 32 + threadIdx.x;
    int r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int r = r0 + i;
        if (r < rows && c < cols) tile[i][threadIdx.x] = in[(size_t)r * cols + c];
    }
    __syncthreads();
    int orow0 = blockIdx.x * 32;   // output row index = input col
    int oc = r0 + threadIdx.x;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int orow = orow0 + i;
        if (orow < cols && oc < rows) out[(size_t)orow * rows + oc] = tile[threadIdx.x][i];
    }
}

// W16[n,k] = half(q - z) * half(s), fp16 multiply (KERNEL_dequant OUT_TYPE=0 semantics)
__global__ void k_dequant_k_major(const uint32_t* __restrict__ qw, const uint8_t* __restrict__ qz,
                                  const __half* __restrict__ sc, __half* __restrict__ out, int N, int K8,
                                  int G8) {
    int n = blockIdx.x;
    int groups = K8 / G8;
    for (int k8 = threadIdx.x; k8 < K8; k8 += blockDim.x) {
        uint32_t w = qw[(size_t)n * K8 + k8];
        int g = k8 / G8;
        __half s = sc[(size_t)n * groups + g];
        int z = qz[(size_t)n * groups + g];
        __half o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            int q = (w >> km_nibble_shift(i)) & 0xF;
            o[i] = __hmul(__int2half_rn(q - z), s);
        }
        *reinterpret_cast<uint4*>(out + (size_t)n * K8 * 8 + (size_t)k8 * 8) = *reinterpret_cast<uint4*>(o);
    }
}

// ---- ZLW4 packer: one thread per packed weight word; a few threads per block also write the meta ----
__global__ void k_w4_pack(const uint32_t* __restrict__ qw, const uint8_t* __restrict__ qz,
                          const __half* __restrict__ sc, const int32_t* __restrict__ row_map,
                          uint8_t* __restrict__ packed, int N, int K, int sym, int variant) {
    const int G = K / kW4GroupK;
    const int K8 = K / 8;
    const int st = blockIdx.x;       // super tile (32 rows)
    const int gi = blockIdx.y;       // k-group
    uint8_t* blk = packed + ((size_t)st * G + gi) * kW4BlockBytes;
    // 512 weight words per block: index = ((tt*2+hh)*32 + lane)*4 + jj
    for (int idx = threadIdx.x; idx < 512; idx += blockDim.x) {
        int jj = idx & 3;
        int lane = (idx >> 2) & 31;
        int hh = (idx >> 7) & 1;
        int tt = idx >> 8;
        int g = lane >> 2, t = lane & 3;
        int j = hh * 4 + jj;
        uint32_t word = 0;
#pragma unroll
        for (int slot = 0; slot < 8; ++slot) {
            int prow, k, shift;
            if (variant == kW4VariantInt) {
                prow = st * 32 + tt * 16 + g + ((slot & 1) ? 8 : 0);
                k = gi * kW4GroupK + w4i_phys_k(t, j >> 1, j & 1, slot >> 1);
                shift = 4 * slot;
            } else {
                prow = st * 32 + tt * 16 + g + (((slot >> 1) & 1) ? 8 : 0);
                k = gi * kW4GroupK + w4_phys_k(t, j, slot >> 2, slot & 1);
                shift = w4_slot_shift(slot);
            }
            int srow = row_map ? row_map[prow] : prow;
            uint32_t src = qw[(size_t)srow * K8 + (k >> 3)];
            uint32_t q = (src >> km_nibble_shift(k & 7)) & 0xFu;
            word |= q << shift;
        }
        reinterpret_cast<uint32_t*>(blk)[idx] = word;
    }
    // meta: 16 (tt,g) entries
    if (threadIdx.x < 16) {
        int tt = threadIdx.x >> 3, g = threadIdx.x & 7;
        int prow0 = st * 32 + tt * 16 + g;
        int r0 = row_map ? row_map[prow0] : prow0;
        int r1 = row_map ? row_map[prow0 + 8] : prow0 + 8;
        __half2 s2 = __halves2half2(sc[(size_t)r0 * G + gi], sc[(size_t)r1 * G + gi]);
        reinterpret_cast<__half2*>(blk + kW4ScaleOff)[threadIdx.x] = s2;
        uint32_t z0 = (sym || !qz) ? 8u : qz[(size_t)r0 * G + gi];
        uint32_t z1 = (sym || !qz) ? 8u : qz[(size_t)r1 * G + gi];
        blk[kW4ZeroOff + threadIdx.x] = (uint8_t)((z0 & 0xF) | ((z1 & 0xF) << 4));
    }
}

__global__ void k_w4_unpack(const uint8_t* __restrict__ packed, uint32_t* __restrict__ qw,
                            uint8_t* __restrict__ qz, __half* __restrict__ sc, int N, int K, int variant) {
    const int G = K / kW4GroupK;
    const int K8 = K / 8;
    const int st = blockIdx.x, gi = blockIdx.y;
    const uint8_t* blk = packed + ((size_t)st * G + gi) * kW4BlockBytes;
    // one thread per (row in 32, k-word in 16)
    for (int idx = threadIdx.x; idx < 32 * 16; idx += blockDim.x) {
        int rr = idx >> 4, kw = idx & 15;
        int tt = rr >> 4, r16 = rr & 15, g = r16 & 7, up = r16 >> 3;
        uint32_t out = 0;
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            int kin = kw * 8 + kk;                 // k within the 128-group
            int t, j, shift;
            if (variant == kW4VariantInt) {
                // kin = t*32 + js*8 + p*4 + i ; word index j = 2*js + p ; nibble = 2*i + up
                t = kin >> 5;
                j = (((kin >> 3) & 3) << 1) | ((kin >> 2) & 1);
                shift = 4 * (((kin & 3) << 1) | up);
            } else {
                // invert w4_phys_k: kin = (u/8)*32 + t*8 + (u%8)
                t = (kin >> 3) & 3;
                int u = ((kin >> 5) << 3) | (kin & 7);
                j = u >> 2;
                int r = (u >> 1) & 1, e = u & 1;
                shift = w4_slot_shift((r << 2) | (up << 1) | e);
            }
            int lane = g * 4 + t;
            int hh = j >> 2, jj = j & 3;
            uint32_t word = reinterpret_cast<const uint32_t*>(blk)[((tt * 2 + hh) * 32 + lane) * 4 + jj];
            uint32_t q = (word >> shift) & 0xFu;
            out |= q << km_nibble_shift(kk);
        }
        qw[(size_t)(st * 32 + rr) * K8 + gi * 16 + kw] = out;
    }
    if (threadIdx.x < 32) {
        int rr = threadIdx.x;
        int tt = rr >> 4, r16 = rr & 15, g = r16 & 7, up = r16 >> 3;
        __half2 s2 = reinterpret_cast<const __half2*>(blk + kW4ScaleOff)[tt * 8 + g];
        sc[(size_t)(st * 32 + rr) * G + gi] = up ? __high2half(s2) : __low2half(s2);
        uint8_t zz = blk[kW4ZeroOff + tt * 8 + g];
        qz[(size_t)(st * 32 + rr) * G + gi] = up ? (zz >> 4) : (zz & 0xF);
    }
}

}  // namespace zl

using namespace zl;

static inline unsigned blocks_for(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

extern "C" int zl_gptq_shuffle(uint32_t* qweight, const int32_t* q_perm, uint32_t* scratch, int K, int N,
                               zl_stream_t stream) {
    ZL_CHECK_ARG(qweight && K > 0 && N > 0 && K % 8 == 0);
    size_t n = (size_t)(K / 8) * N;
    if (q_perm) {
        ZL_CHECK_ARG(scratch != nullptr);
        dim3 grid(cdiv(N, 128), K / 8);
        k_make_sequential<<<grid, 128, 0, stream>>>(qweight, scratch, q_perm, K / 8, N);
        ZL_CHECK_LAUNCH();
        ZL_CHECK_CUDA(cudaMemcpyAsync(qweight, scratch, n * 4, cudaMemcpyDeviceToDevice, stream));
    }
    k_shuffle_words<<<blocks_for(n, 256), 256, 0, stream>>>(qweight, n);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_gptq_increase_zero(uint32_t* qzeros, size_t n_words, zl_stream_t stream) {
    ZL_CHECK_ARG(qzeros && n_words > 0);
    k_inc_zero<<<blocks_for(n_words, 256), 256, 0, stream>>>(qzeros, n_words);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_gptq_subtract8(uint32_t* words, size_t n_words, zl_stream_t stream) {
    ZL_CHECK_ARG(words && n_words > 0);
    k_sub8<<<blocks_for(n_words, 256), 256, 0, stream>>>(words, n_words);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_q4_to_q8(const uint32_t* in, uint8_t* out, size_t n_words, zl_stream_t stream) {
    ZL_CHECK_ARG(in && out && n_words > 0);
    k_q4_to_q8<<<blocks_for(n_words, 256), 256, 0, stream>>>(in, reinterpret_cast<uint2*>(out), n_words);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_awq_un_shuffle(uint32_t* qzeros, int rows, int cols, zl_stream_t stream) {
    ZL_CHECK_ARG(qzeros && rows > 0 && cols > 0);
    size_t n = (size_t)rows * cols;
    k_awq_un_shuffle<<<blocks_for(n, 256), 256, 0, stream>>>(qzeros, n);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_awq_shuffle(const uint32_t* in, uint32_t* out, int K, int N, int use_exllama,
                              zl_stream_t stream) {
    ZL_CHECK_ARG(in && out && K > 0 && N > 0 && K % 8 == 0 && N % 8 == 0);
    dim3 grid(cdiv(N / 8, 64), K / 8);
    k_awq_shuffle<<<grid, 64, 0, stream>>>(in, out, K / 8, N / 8, use_exllama);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_transpose_2d(const void* in, void* out, int rows, int cols, int elem_bytes,
                               zl_stream_t stream) {
    ZL_CHECK_ARG(in && out && rows > 0 && cols > 0);
    dim3 grid(cdiv(cols, 32), cdiv(rows, 32)), block(32, 8);
    if (elem_bytes == 4)
        k_transpose<uint32_t><<<grid, block, 0, stream>>>((const uint32_t*)in, (uint32_t*)out, rows, cols);
    else if (elem_bytes == 2)
        k_transpose<uint16_t><<<grid, block, 0, stream>>>((const uint16_t*)in, (uint16_t*)out, rows, cols);
    else if (elem_bytes == 1)
        k_transpose<uint8_t><<<grid, block, 0, stream>>>((const uint8_t*)in, (uint8_t*)out, rows, cols);
    else
        ZL_CHECK_SUPPORTED(elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_gptq_dequant_k_major(const uint32_t* qweight_km, const uint8_t* qzeros_km,
                                       const void* scales_km, void* out_f16, int N, int K, int group_size,
                                       zl_stream_t stream) {
    ZL_CHECK_ARG(qweight_km && qzeros_km && scales_km && out_f16 && N > 0 && K > 0);
    ZL_CHECK_ARG(K % 8 == 0 && group_size % 8 == 0 && K % group_size == 0);
    k_dequant_k_major<<<N, 128, 0, stream>>>(qweight_km, qzeros_km, (const __half*)scales_km, (__half*)out_f16,
                                             N, K / 8, group_size / 8);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" size_t zl_w4_packed_bytes(int N, int K, int group_size) {
    if (N <= 0 || K <= 0 || group_size != kW4GroupK || N % 32 || K % kW4GroupK) return 0;
    return (size_t)(N / 32) * (K / kW4GroupK) * kW4BlockBytes;
}

extern "C" int zl_w4_pack_v(const uint32_t* qweight_km, const uint8_t* qzeros_km, const void* scales_km,
                            const int32_t* row_map, void* packed, int N, int K, int group_size, int sym, int variant,
                            zl_stream_t stream) {
    ZL_CHECK_ARG(qweight_km && scales_km && packed && N > 0 && K > 0);
    ZL_CHECK_ARG(sym || qzeros_km);
    ZL_CHECK_SUPPORTED(group_size == kW4GroupK);
    ZL_CHECK_SUPPORTED(N % 32 == 0 && K % kW4GroupK == 0);
    dim3 grid(N / 32, K / kW4GroupK);
    ZL_CHECK_ARG(variant == kW4VariantHalf || variant == kW4VariantInt);
    k_w4_pack<<<grid, 256, 0, stream>>>(qweight_km, qzeros_km, (const __half*)scales_km, row_map,
                                        (uint8_t*)packed, N, K, sym, variant);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_w4_pack(const uint32_t* qweight_km, const uint8_t* qzeros_km, const void* scales_km,
                          const int32_t* row_map, void* packed, int N, int K, int group_size, int sym,
                          zl_stream_t stream) {
    return zl_w4_pack_v(qweight_km, qzeros_km, scales_km, row_map, packed, N, K, group_size, sym, kW4VariantHalf, stream);
}

extern "C" int zl_w4_unpack_v(const void* packed, uint32_t* qweight_km, uint8_t* qzeros_km, void* scales_km,
                              int N, int K, int group_size, int variant, zl_stream_t stream) {
    ZL_CHECK_ARG(packed && qweight_km && qzeros_km && scales_km && N > 0 && K > 0);
    ZL_CHECK_SUPPORTED(group_size == kW4GroupK && N % 32 == 0 && K % kW4GroupK == 0);
    dim3 grid(N / 32, K / kW4GroupK);
    ZL_CHECK_ARG(variant == kW4VariantHalf || variant == kW4VariantInt);
    k_w4_unpack<<<grid, 256, 0, stream>>>((const uint8_t*)packed, qweight_km, qzeros_km, (__half*)scales_km, N,
                                          K, variant);
    ZL_CHECK_LAUNCH();
    return ZL_OK;
}

extern "C" int zl_w4_unpack(const void* packed, uint32_t* qweight_km, uint8_t* qzeros_km, void* scales_km,
                            int N, int K, int group_size, zl_stream_t stream) {
    return zl_w4_unpack_v(packed, qweight_km, qzeros_km, scales_km, N, K, group_size, kW4VariantHalf, stream);
}

// ---- act-order activation permute: y[m, i] = x[m, perm[i]] (nn::gptq::permute_input, gptq/utils.cu:322-398) -------
// For the GEMM routes whose activation tiles arrive by TMA and so cannot gather (the integer kernel gathers while it
// stages).  8 output columns per thread: two 16-byte index loads, eight 2-byte gathers, one 16-byte store.
namespace zl {
__global__ void k_gather_cols_16(const uint16_t* __restrict__ x, int ldx, const int32_t* __restrict__ perm,
                                 uint16_t* __restrict__ y, int K) {
    pdl_trigger();
    const int c8 = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = c8 * 8 < K;
    int4 a = make_int4(0, 0, 0, 0), b = a;
    if (live) {   // the permutation is a constant: load it before waiting on the producer of x
        a = __ldg(reinterpret_cast<const int4*>(perm) + 2 * c8);
        b = __ldg(reinterpret_cast<const int4*>(perm) + 2 * c8 + 1);
    }
    pdl_wait();
    if (!live) return;
    const uint16_t* xr = x + (size_t)blockIdx.y * ldx;
    uint4 o;
    o.x = (uint32_t)xr[a.x] | ((uint32_t)xr[a.y] << 16);
    o.y = (uint32_t)xr[a.z] | ((uint32_t)xr[a.w] << 16);
    o.z = (uint32_t)xr[b.x] | ((uint32_t)xr[b.y] << 16);
    o.w = (uint32_t)xr[b.z] | ((uint32_t)xr[b.w] << 16);
    *reinterpret_cast<uint4*>(y + (size_t)blockIdx.y * K + c8 * 8) = o;
}
}  // namespace zl

extern "C" int zl_gather_cols_16(const void* x, int ldx, const int32_t* perm, void* y, int M, int K, int pdl,
                                 zl_stream_t stream) {
    ZL_CHECK_ARG(x && perm && y && M > 0 && M <= 65535 && K > 0 && K % 8 == 0 && ldx >= K && ldx % 8 == 0);
    ZL_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(perm) & 15) == 0);
    const dim3 grid(zl::cdiv(K / 8, 128), M);
    ZL_CHECK_CUDA(zl::launch(zl::k_gather_cols_16, grid, dim3(128), 0, (cudaStream_t)stream, pdl != 0,
                             (const uint16_t*)x, ldx, perm, (uint16_t*)y, K));
    return ZL_OK;
}
