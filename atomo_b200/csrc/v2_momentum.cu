// Momentum correction for top-k on the overlapped, sharded bf16 engine (sm_90a): the apply pass of ONE backward group
// (Deep Gradient Compression, Lin et al. 2018).
//
// With momentum_correction the workers, not the parameter server, apply momentum and weight decay, before the
// gradient is sparsified; the PS runs plain SGD.  Each worker keeps an fp32 momentum u per weight element (`mom`, the
// physical order of wshadow, the offsets of the error-feedback residual e) and per vector element (`vmom`, the order
// of vgrads).  On the encode stream, once the group's gradients exist, this launch takes the place of
// v2_ef_apply_kernel:
//
//   weights   d = wd > 0 ? g + wd w : g        (g the bf16 gradient autograd wrote, w the bf16 weight in wshadow that
//             u = m u + d                       this step's forward used: the group's PS waits for this push before
//             s = nesterov ? d + m u : u        it publishes new weights)
//             A = s + e;  bf16(A) into the gradient buffer in place, e = A - bf16(A)
//   vectors   d = wd > 0 ? v + wd p : v,  u = m u + d,  v = nesterov ? d + m u : u   (vgrads in place, p = vparams)
//
// The top-k encode then runs on bf16(A) unchanged; its masking variant (v2_topk_encode_mc_kernel) also stores u = 0 for
// every kept entry (momentum-factor masking).  Vectors travel exactly and are not masked.  Every sum and product is a
// named round-to-nearest intrinsic, so an fp32 oracle matches the pass bit for bit.  Bandwidth bound, with the chunk
// geometry and 16-byte accesses of v2_ef_apply_kernel: 2 + 4 + 4 bytes read and 2 + 4 + 4 written per weight element,
// plus 2 read for w when wd > 0.
#include "v2_common.cuh"
#include "v2_momentum.cuh"

namespace atomo {
namespace v2 {

constexpr int MC_THREADS = 256;

// Blocks [0, nw) take the group's weight chunks, the rest its vector chunks (v2_accum_add_kernel's split).
__global__ void __launch_bounds__(MC_THREADS) v2_mc_apply_kernel(const EfChunk* wchunks, int nw, const EfChunk* vchunks,
                                                                 const long long* gptr, const __nv_bfloat16* wshadow,
                                                                 float* mom, float* residual, float* vgrads,
                                                                 const float* vparams, float* vmom, float m, float wd,
                                                                 int nesterov) {
  const bool use_wd = wd > 0.f, nest = nesterov != 0;
  if ((int)blockIdx.x < nw) {
    const EfChunk c = wchunks[blockIdx.x];
    __nv_bfloat16* g = reinterpret_cast<__nv_bfloat16*>(gptr[c.widx]) + c.start;
    const __nv_bfloat16* w = wshadow + c.w_off + c.start;
    float* u = mom + c.w_off + c.start;
    float* e = residual + c.w_off + c.start;
    // mom and the residual share wshadow's offsets (multiples of 64 elements) and chunks start on multiples of 8, so
    // only a gradient buffer that autograd hands over unaligned takes the scalar path
    const bool vec = ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(u) |
                       reinterpret_cast<uintptr_t>(e)) & 15) == 0;
    const int nv = vec ? (c.count >> 3) : 0;
    for (int v = threadIdx.x; v < nv; v += blockDim.x) {
      const uint4 gw = *reinterpret_cast<const uint4*>(g + 8 * v);
      float d[8] = {bf16_lo(gw.x), bf16_hi(gw.x), bf16_lo(gw.y), bf16_hi(gw.y),
                    bf16_lo(gw.z), bf16_hi(gw.z), bf16_lo(gw.w), bf16_hi(gw.w)};
      if (use_wd) {
        const uint4 ww = __ldg(reinterpret_cast<const uint4*>(w + 8 * v));
        const float x[8] = {bf16_lo(ww.x), bf16_hi(ww.x), bf16_lo(ww.y), bf16_hi(ww.y),
                            bf16_lo(ww.z), bf16_hi(ww.z), bf16_lo(ww.w), bf16_hi(ww.w)};
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = __fadd_rn(d[i], __fmul_rn(wd, x[i]));
      }
      const float4 u0 = reinterpret_cast<const float4*>(u)[2 * v];
      const float4 u1 = reinterpret_cast<const float4*>(u)[2 * v + 1];
      const float4 e0 = reinterpret_cast<const float4*>(e)[2 * v];
      const float4 e1 = reinterpret_cast<const float4*>(e)[2 * v + 1];
      float uu[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
      float r[8] = {e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w};
      __nv_bfloat16 b[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) r[i] = ef_round(__fadd_rn(mc_step(d[i], uu[i], m, nest), r[i]), b[i]);
      uint32_t o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
        o[i] = (uint32_t)__bfloat16_as_ushort(b[2 * i]) | ((uint32_t)__bfloat16_as_ushort(b[2 * i + 1]) << 16);
      *reinterpret_cast<uint4*>(g + 8 * v) = make_uint4(o[0], o[1], o[2], o[3]);
      reinterpret_cast<float4*>(u)[2 * v] = make_float4(uu[0], uu[1], uu[2], uu[3]);
      reinterpret_cast<float4*>(u)[2 * v + 1] = make_float4(uu[4], uu[5], uu[6], uu[7]);
      reinterpret_cast<float4*>(e)[2 * v] = make_float4(r[0], r[1], r[2], r[3]);
      reinterpret_cast<float4*>(e)[2 * v + 1] = make_float4(r[4], r[5], r[6], r[7]);
    }
    for (int i = (nv << 3) + threadIdx.x; i < c.count; i += blockDim.x) {
      float d = __bfloat162float(g[i]);
      if (use_wd) d = __fadd_rn(d, __fmul_rn(wd, __bfloat162float(w[i])));
      float ui = u[i];
      __nv_bfloat16 b;
      e[i] = ef_round(__fadd_rn(mc_step(d, ui, m, nest), e[i]), b);
      u[i] = ui;
      g[i] = b;
    }
    return;
  }
  const EfChunk c = vchunks[blockIdx.x - nw];
  float* s = vgrads + c.w_off + c.start;
  const float* p = vparams + c.w_off + c.start;
  float* u = vmom + c.w_off + c.start;
  for (int i = threadIdx.x; i < c.count; i += blockDim.x) {
    const float d = use_wd ? __fadd_rn(s[i], __fmul_rn(wd, p[i])) : s[i];
    float ui = u[i];
    s[i] = mc_step(d, ui, m, nest);
    u[i] = ui;
  }
}

extern "C" {

void atomo_v2_launch_mc_apply(const void* wchunks, int nw, const void* vchunks, int nv, const long long* gptr,
                              const void* wshadow, float* mom, float* residual, float* vgrads, const float* vparams,
                              float* vmom, float m, float wd, int nesterov, cudaStream_t stream) {
  if (nw + nv <= 0) return;
  v2_mc_apply_kernel<<<nw + nv, MC_THREADS, 0, stream>>>((const EfChunk*)wchunks, nw, (const EfChunk*)vchunks, gptr,
                                                         (const __nv_bfloat16*)wshadow, mom, residual, vgrads, vparams,
                                                         vmom, m, wd, nesterov);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
