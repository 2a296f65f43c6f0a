// The e4m3 quantisation rule of compute_type float8_float16, defined once for every kernel that quantises (encoder weights at
// load, LayerNorm outputs, attention and GELU outputs).  oracle/fp8_oracle.py mirrors it on the CPU.
//
// Per row (a weight's output channel, or an activation's token over the whole K):
//   scale s = amax / 448 (correctly rounded fp32 division; a row whose amax is 0 gets s = 1 and all-zero codes)
//   code  q = e4m3(x / s)  (correctly rounded division, then round-to-nearest-even with saturation to +-448)
// and a GEMM of two such operands is D[r][n] = s_a[r] s_w[n] sum_k q_a[r][k] q_w[n][k].
#pragma once
#include <stdint.h>

namespace b2w {

constexpr float kE4m3Max = 448.f;

#ifdef __CUDACC__
__device__ __forceinline__ float e4m3_row_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, kE4m3Max) : 1.f; }

// two values -> two e4m3 codes, lo in the low byte (the lower address)
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi, float s) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(__fdiv_rn(hi, s)), "f"(__fdiv_rn(lo, s)));
  return r;
}
// four values -> four codes in memory order
__device__ __forceinline__ uint32_t e4m3x4(float a, float b, float c, float d, float s) {
  return e4m3x2(a, b, s) | (e4m3x2(c, d, s) << 16);
}
#endif

}  // namespace b2w
