// ZLW4: tile-packed int4 weight layout for the W4A16 kernels (DESIGN.md section 3).
//
// The matrix W (N rows = output features, K cols) is cut into blocks of 32 rows x 128 k
// (= one quantization group of the g128 checkpoints).  Blocks are stored [N/32][K/128], each
// block is ONE contiguous 2128-byte record so that a single 1-D bulk-TMA copy (cp.async.bulk)
// brings weights + scales + zeros of a block into shared memory:
//
//   [   0,2048)  weights: [tile tt (2)][half hh (2)][lane (32)] uint4
//                lane = 4*g + t (g = 0..7, t = 0..3) is the mma.sync m16n8k16 lane that will own the
//                data; word j = 4*hh + jj (jj = uint4 component) is the complete A fragment of MMA j:
//                  nibble slots  e0 e1 | e2 e3 | e4 e5 | e6 e7
//                  A registers   a0 a1 | a2 a3 | a4 a5 | a6 a7
//                  row           g     | g+8   | g     | g+8      (within 16-row tile tt)
//                  k (in group)  k(j,0,e)      | k(j,1,e)
//                with k(j,r,e) = w4_phys_k(t, j, r, e): a permutation of the 128 k of the group chosen
//                so that the matching B fragments (activations) of lane (g,t) are 4 x 16-byte
//                contiguous loads.  Slot e_i sits at bit (i>>1)*4 + (i&1)*16, i.e. the word has the
//                reference's "q0 q2 q4 q6 | q1 q3 q5 q7" nibble order (qdq_4.cuh:16-35) and is decoded
//                with the same lop3 0x6400 magic-number trick (q_gemm_k_major.cu:74-98).
//   [2048,2112)  scales : [tt (2)][g (8)] half2 { s[row g], s[row g+8] }
//   [2112,2128)  zeros  : [tt (2)][g (8)] uint8  z[row g] | z[row g+8] << 4   (already +1'd, wrapped)
#pragma once
#include <stdint.h>

namespace zl {

constexpr int kW4GroupK = 128;
constexpr int kW4TileRows = 32;
constexpr int kW4WeightBytes = 2048;
constexpr int kW4ScaleOff = 2048;
constexpr int kW4ZeroOff = 2112;
constexpr int kW4BlockBytes = 2128;

// bit position of natural k index kk (0..7) inside a reference k-major (shuffled) word
__host__ __device__ __forceinline__ int km_nibble_shift(int kk) { return (kk >> 1) * 4 + (kk & 1) * 16; }
// bit position of nibble slot e_i inside a ZLW4 word (same formula, different meaning)
__host__ __device__ __forceinline__ int w4_slot_shift(int slot) { return (slot >> 1) * 4 + (slot & 1) * 16; }
// physical k (0..127 within the group) of MMA j (0..7), register half r (0: k 2t..2t+1, 1: k 2t+8..), element e
__host__ __device__ __forceinline__ int w4_phys_k(int t, int j, int r, int e) {
    int u = j * 4 + r * 2 + e;
    return (u >> 3) * 32 + t * 8 + (u & 7);
}

// ---- ZLW4I: same 2128-byte block, nibble order for the exact-integer kernel (IMMA m16n8k32) -------------
//   word wi = 2*j + p of lane (g,t) (j = MMA k-step 0..3, p = register pair 0/1) holds, for byte i = 0..3:
//     nibble 2i   = W[row g  ][k = t*32 + j*8 + p*4 + i]        -> A reg a_{2p}   = w & 0x0f0f0f0f
//     nibble 2i+1 = W[row g+8][same k]                           -> A reg a_{2p+1} = w & 0xf0f0f0f0 (value * 16)
//   i.e. k is in NATURAL order inside the group, so the matching B fragments (int8 activation pieces) of a
//   lane are 32 contiguous bytes.  Meta (scales / zeros) as in ZLW4.
enum { kW4VariantHalf = 0, kW4VariantInt = 1 };
__host__ __device__ __forceinline__ int w4i_phys_k(int t, int j, int pp, int i) { return t * 32 + j * 8 + pp * 4 + i; }

}  // namespace zl
