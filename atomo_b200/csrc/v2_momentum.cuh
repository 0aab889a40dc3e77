// Worker-side heavy-ball momentum of the bf16 engine, shared by momentum correction (v2_momentum.cu) and Signum
// (v2_signum.cu): one definition, so that both codes and their fp32 oracles round the same way.
#pragma once
#include <cuda_runtime.h>

namespace atomo {
namespace v2 {

// u <- m u + d, returns the direction s; d already carries weight decay
__device__ __forceinline__ float mc_step(float d, float& u, float m, bool nesterov) {
  u = __fadd_rn(__fmul_rn(m, u), d);
  return nesterov ? __fadd_rn(d, __fmul_rn(m, u)) : u;
}

}  // namespace v2
}  // namespace atomo
