// bf16 gradient loaders of the bucketed dense codes (v2_sign.cu, v2_fp8.cu).
#pragma once
#include "v2_common.cuh"

namespace atomo {
namespace v2 {

// bf16 subnormals read as signed zero, by bit operations: the code (and codings/sign.py) does not depend on how the
// compiler's flush-to-zero treats them in the comparisons and the fp64 conversions below
__device__ __forceinline__ float sign_ftz(float x) {
  const uint32_t u = __float_as_uint(x);
  return __uint_as_float((u & 0x7f800000u) ? u : (u & 0x80000000u));
}

// elements 8c .. 8c+7 of a bucket, 0 past blen: one 16-byte load for the first nch (aligned, whole) chunks, else
// element loads
__device__ __forceinline__ void sign_load8(const __nv_bfloat16* src, int c, int nch, int blen, float (&x)[8]) {
  if (c < nch) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src) + c);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { x[2 * i] = sign_ftz(bf16_lo(w[i])); x[2 * i + 1] = sign_ftz(bf16_hi(w[i])); }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = 8 * c + i;
      x[i] = e < blen ? sign_ftz(__bfloat162float(src[e])) : 0.f;
    }
  }
}

}  // namespace v2
}  // namespace atomo
