// The int8 KV cache's row quantisation: int8_op::quant_calc_scale(x, 127, 128) of the reference
// (src/nn/quant/int8/quant_kernel.cu:15-47) for one (token, kv head) row of d values with absolute maximum amax.
//   code  = uint8(128 + nearbyint(x * (127 / amax)))
//   scale = amax / 127
// Every kernel that writes cache codes or scales goes through these three functions, so the bytes do not depend on
// which route wrote them.  A row whose amax is 0 keeps the reference's behaviour: 127 / 0 = inf, 0 * inf = NaN, and the
// float -> u8 conversion of NaN gives 0; its scale is 0, so it decodes to 0 whatever the code.
#pragma once
#include <cstdint>

namespace zl {

__device__ __forceinline__ float kv8_row_mul(float amax) { return 127.0f / amax; }
__device__ __forceinline__ uint8_t kv8_code(float x, float mul) { return (uint8_t)(128.f + nearbyintf(x * mul)); }
__device__ __forceinline__ float kv8_row_scale(float amax) { return amax / 127.0f; }

}  // namespace zl
