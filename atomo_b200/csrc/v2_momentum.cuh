// Worker-side momentum of the bf16 engine, shared by momentum correction (v2_momentum.cu), Signum and Distributed Lion
// (v2_signum.cu) and the PS kernels' Lion (v2_ps_common.cuh): one definition of each rule, so that every code and its
// fp32 oracle round the same way.
#pragma once
#include <cuda_runtime.h>

namespace atomo {
namespace v2 {

// u <- m u + d, returns the direction s; d already carries weight decay
__device__ __forceinline__ float mc_step(float d, float& u, float m, bool nesterov) {
  u = __fadd_rn(__fmul_rn(m, u), d);
  return nesterov ? __fadd_rn(d, __fmul_rn(m, u)) : u;
}

// Lion (Chen et al. 2023), as two lines: the direction c = b1 m + (1 - b1) g, then the momentum m <- b2 m + (1 - b2) g.
// Every operation is rounded on its own (no contraction) and 1 - b is formed in fp32.
__device__ __forceinline__ float lion_direction(float g, float m, float b1) {
  return __fadd_rn(__fmul_rn(b1, m), __fmul_rn(__fsub_rn(1.f, b1), g));
}
__device__ __forceinline__ float lion_momentum(float g, float m, float b2) {
  return __fadd_rn(__fmul_rn(b2, m), __fmul_rn(__fsub_rn(1.f, b2), g));
}

}  // namespace v2
}  // namespace atomo
