// wgmma.mma_async wrappers (m64 x N, N = 32 / 64 / 128 / 256) used by w4a16_tc.cu and w8_tc.cu:
//   wg_f16_rs  : f16 x f16 -> f32, A (64 x 16) from registers, B (N x 16, K-major) from shared memory
//   wg_s8_ss   : s8 x s8 -> s32 (exact), both operands from shared memory (K-major)
//   wg_e4m3_ss : e4m3 x e4m3 -> f32 (N <= 128), both operands from shared memory (K-major)
// `accum` = 0 overwrites the accumulators, otherwise the products are added to them.
#pragma once
#include <stdint.h>

namespace zl {

template <int N>
__device__ __forceinline__ void wg_f16_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accum);
template <int N>
__device__ __forceinline__ void wg_s8_ss(int (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum);
template <int N>
__device__ __forceinline__ void wg_e4m3_ss(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum);

// eight accumulator operands d[i .. i + 7] with constraint C
#define ZL_ACC8(C, i) C(d[i]), C(d[i + 1]), C(d[i + 2]), C(d[i + 3]), C(d[i + 4]), C(d[i + 5]), C(d[i + 6]), C(d[i + 7])

// accumulator register lists {%0, ..., %(N/2 - 1)}
#define ZL_D32 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}"
#define ZL_D64 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"
#define ZL_D128 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"
#define ZL_D256 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}"
template <> __device__ __forceinline__ void wg_f16_rs<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\nwgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 " ZL_D32
                 ", {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n}"
                 : ZL_ACC8("+f", 0), ZL_ACC8("+f", 8) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_s8_ss<32>(int (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\nwgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 " ZL_D32
                 ", %16, %17, p;\n}"
                 : ZL_ACC8("+r", 0), ZL_ACC8("+r", 8) : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_e4m3_ss<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\nwgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 " ZL_D32
                 ", %16, %17, p, 1, 1;\n}"
                 : ZL_ACC8("+f", 0), ZL_ACC8("+f", 8) : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_f16_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\nwgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " ZL_D64
                 ", {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n}"
                 : ZL_ACC8("+f", 0), ZL_ACC8("+f", 8), ZL_ACC8("+f", 16), ZL_ACC8("+f", 24) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_s8_ss<64>(int (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\nwgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 " ZL_D64
                 ", %32, %33, p;\n}"
                 : ZL_ACC8("+r", 0), ZL_ACC8("+r", 8), ZL_ACC8("+r", 16), ZL_ACC8("+r", 24) : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_e4m3_ss<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\nwgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 " ZL_D64
                 ", %32, %33, p, 1, 1;\n}"
                 : ZL_ACC8("+f", 0), ZL_ACC8("+f", 8), ZL_ACC8("+f", 16), ZL_ACC8("+f", 24) : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_f16_rs<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\nwgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " ZL_D128
                 ", {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n}"
                 : ZL_ACC8("+f", 0), ZL_ACC8("+f", 8), ZL_ACC8("+f", 16), ZL_ACC8("+f", 24), ZL_ACC8("+f", 32), ZL_ACC8("+f", 40), ZL_ACC8("+f", 48), ZL_ACC8("+f", 56) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_s8_ss<128>(int (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\nwgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 " ZL_D128
                 ", %64, %65, p;\n}"
                 : ZL_ACC8("+r", 0), ZL_ACC8("+r", 8), ZL_ACC8("+r", 16), ZL_ACC8("+r", 24), ZL_ACC8("+r", 32), ZL_ACC8("+r", 40), ZL_ACC8("+r", 48), ZL_ACC8("+r", 56) : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_e4m3_ss<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\nwgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 " ZL_D128
                 ", %64, %65, p, 1, 1;\n}"
                 : ZL_ACC8("+f", 0), ZL_ACC8("+f", 8), ZL_ACC8("+f", 16), ZL_ACC8("+f", 24), ZL_ACC8("+f", 32), ZL_ACC8("+f", 40), ZL_ACC8("+f", 48), ZL_ACC8("+f", 56) : "l"(adesc), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_f16_rs<256>(float (&d)[128], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %133, 0;\nwgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " ZL_D256
                 ", {%128,%129,%130,%131}, %132, p, 1, 1, 0;\n}"
                 : ZL_ACC8("+f", 0), ZL_ACC8("+f", 8), ZL_ACC8("+f", 16), ZL_ACC8("+f", 24), ZL_ACC8("+f", 32), ZL_ACC8("+f", 40), ZL_ACC8("+f", 48), ZL_ACC8("+f", 56), ZL_ACC8("+f", 64), ZL_ACC8("+f", 72), ZL_ACC8("+f", 80), ZL_ACC8("+f", 88), ZL_ACC8("+f", 96), ZL_ACC8("+f", 104), ZL_ACC8("+f", 112), ZL_ACC8("+f", 120) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum));
}
template <> __device__ __forceinline__ void wg_s8_ss<256>(int (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\nwgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 " ZL_D256
                 ", %128, %129, p;\n}"
                 : ZL_ACC8("+r", 0), ZL_ACC8("+r", 8), ZL_ACC8("+r", 16), ZL_ACC8("+r", 24), ZL_ACC8("+r", 32), ZL_ACC8("+r", 40), ZL_ACC8("+r", 48), ZL_ACC8("+r", 56), ZL_ACC8("+r", 64), ZL_ACC8("+r", 72), ZL_ACC8("+r", 80), ZL_ACC8("+r", 88), ZL_ACC8("+r", 96), ZL_ACC8("+r", 104), ZL_ACC8("+r", 112), ZL_ACC8("+r", 120) : "l"(adesc), "l"(bdesc), "r"(accum));
}
#undef ZL_D32
#undef ZL_D64
#undef ZL_D128
#undef ZL_D256
#undef ZL_ACC8

}  // namespace zl
