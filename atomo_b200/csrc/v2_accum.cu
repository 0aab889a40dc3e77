// Gradient accumulation on the overlapped, sharded bf16 engine (sm_90a): the two passes of ONE backward group.
//
// With accumulate_steps = N a step runs N micro-batches, and only the last one codes and pushes.  Each worker keeps
// an fp32 accumulator per weight element (`acc`, the physical order of wshadow) and per vector element (`vacc`, the
// order of vgrads), both zero at every step boundary:
//
//   v2_accum_add_kernel    micro-batches 1 .. N-1, on the encode stream once the group's gradients exist:
//                          acc += g (the first micro-batch stores), with g autograd's bf16 gradient buffer read
//                          through this micro-batch's pointer table; vacc += vgrads, then vgrads = 0 for the next
//                          micro-batch's backward.  The engine then releases the gradient buffers.
//   v2_accum_fold_kernel   micro-batch N, before the group's encode: A = (acc + g) * fp32(1/N), with error feedback
//                          A += e; bf16(A) written back in place into the last micro-batch's gradient buffer (so the
//                          encoders, --code-stats and the EF epilogues read it unchanged), A - bf16(A) into the
//                          residual (error feedback only; it replaces v2_ef_apply_kernel for the group), acc = 0;
//                          vgrads = (vacc + vgrads) * fp32(1/N), vacc = 0.
//
// Every sum and product is a named round-to-nearest intrinsic, in micro-batch order, so an fp32 oracle matches the
// passes bit for bit.  Bandwidth bound, with the chunk geometry and 16-byte accesses of v2_ef_apply_kernel: the add
// reads 2 + 4 bytes and writes 4 per weight element (2 + 4 for the first micro-batch), the fold reads 2 + 4 and
// writes 2 + 4 (4 more of each with error feedback).
#include "v2_common.cuh"

namespace atomo {
namespace v2 {

constexpr int ACC_THREADS = 256;

__device__ __forceinline__ void unpack8(const uint4 w, float (&x)[8]) {
  x[0] = bf16_lo(w.x); x[1] = bf16_hi(w.x); x[2] = bf16_lo(w.y); x[3] = bf16_hi(w.y);
  x[4] = bf16_lo(w.z); x[5] = bf16_hi(w.z); x[6] = bf16_lo(w.w); x[7] = bf16_hi(w.w);
}

// Blocks [0, nw) take the weight chunks, the rest the vector chunks of the group.
__global__ void __launch_bounds__(ACC_THREADS) v2_accum_add_kernel(const EfChunk* wchunks, int nw,
                                                                   const EfChunk* vchunks, const long long* gptr,
                                                                   float* acc, float* vacc, float* vgrads,
                                                                   int first) {
  if ((int)blockIdx.x < nw) {
    const EfChunk c = wchunks[blockIdx.x];
    const __nv_bfloat16* g = reinterpret_cast<const __nv_bfloat16*>(gptr[c.widx]) + c.start;
    float* a = acc + c.w_off + c.start;
    const bool vec = ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(a)) & 15) == 0;
    const int nv = vec ? (c.count >> 3) : 0;
    for (int v = threadIdx.x; v < nv; v += blockDim.x) {
      float x[8];
      unpack8(*reinterpret_cast<const uint4*>(g + 8 * v), x);
      if (!first) {
        const float4 a0 = reinterpret_cast<const float4*>(a)[2 * v];
        const float4 a1 = reinterpret_cast<const float4*>(a)[2 * v + 1];
        const float s[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = __fadd_rn(s[i], x[i]);
      }
      reinterpret_cast<float4*>(a)[2 * v] = make_float4(x[0], x[1], x[2], x[3]);
      reinterpret_cast<float4*>(a)[2 * v + 1] = make_float4(x[4], x[5], x[6], x[7]);
    }
    for (int i = (nv << 3) + threadIdx.x; i < c.count; i += blockDim.x) {
      const float x = __bfloat162float(g[i]);
      a[i] = first ? x : __fadd_rn(a[i], x);
    }
    return;
  }
  const EfChunk c = vchunks[blockIdx.x - nw];
  float* s = vgrads + c.w_off + c.start;
  float* a = vacc + c.w_off + c.start;
  for (int i = threadIdx.x; i < c.count; i += blockDim.x) {
    a[i] = first ? s[i] : __fadd_rn(a[i], s[i]);
    s[i] = 0.f;
  }
}

__global__ void __launch_bounds__(ACC_THREADS) v2_accum_fold_kernel(const EfChunk* wchunks, int nw,
                                                                    const EfChunk* vchunks, const long long* gptr,
                                                                    float* acc, float* vacc, float* vgrads,
                                                                    float inv_n, float* residual) {
  if ((int)blockIdx.x < nw) {
    const EfChunk c = wchunks[blockIdx.x];
    __nv_bfloat16* g = reinterpret_cast<__nv_bfloat16*>(gptr[c.widx]) + c.start;
    float* a = acc + c.w_off + c.start;
    float* e = residual ? residual + c.w_off + c.start : nullptr;
    // the residual shares the accumulator's offsets, so its alignment is the accumulator's
    const bool vec = ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(a)) & 15) == 0;
    const int nv = vec ? (c.count >> 3) : 0;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int v = threadIdx.x; v < nv; v += blockDim.x) {
      float x[8];
      unpack8(*reinterpret_cast<const uint4*>(g + 8 * v), x);
      const float4 a0 = reinterpret_cast<const float4*>(a)[2 * v];
      const float4 a1 = reinterpret_cast<const float4*>(a)[2 * v + 1];
      const float s[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] = __fmul_rn(__fadd_rn(s[i], x[i]), inv_n);
      __nv_bfloat16 b[8];
      if (e) {
        const float4 e0 = reinterpret_cast<const float4*>(e)[2 * v];
        const float4 e1 = reinterpret_cast<const float4*>(e)[2 * v + 1];
        float r[8] = {e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) r[i] = ef_round(__fadd_rn(x[i], r[i]), b[i]);
        reinterpret_cast<float4*>(e)[2 * v] = make_float4(r[0], r[1], r[2], r[3]);
        reinterpret_cast<float4*>(e)[2 * v + 1] = make_float4(r[4], r[5], r[6], r[7]);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) b[i] = __float2bfloat16_rn(x[i]);
      }
      uint32_t w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
        w[i] = (uint32_t)__bfloat16_as_ushort(b[2 * i]) | ((uint32_t)__bfloat16_as_ushort(b[2 * i + 1]) << 16);
      *reinterpret_cast<uint4*>(g + 8 * v) = make_uint4(w[0], w[1], w[2], w[3]);
      reinterpret_cast<float4*>(a)[2 * v] = zero;
      reinterpret_cast<float4*>(a)[2 * v + 1] = zero;
    }
    for (int i = (nv << 3) + threadIdx.x; i < c.count; i += blockDim.x) {
      float x = __fmul_rn(__fadd_rn(a[i], __bfloat162float(g[i])), inv_n);
      __nv_bfloat16 b;
      if (e) e[i] = ef_round(__fadd_rn(x, e[i]), b);
      else b = __float2bfloat16_rn(x);
      g[i] = b;
      a[i] = 0.f;
    }
    return;
  }
  const EfChunk c = vchunks[blockIdx.x - nw];
  float* s = vgrads + c.w_off + c.start;
  float* a = vacc + c.w_off + c.start;
  for (int i = threadIdx.x; i < c.count; i += blockDim.x) {
    s[i] = __fmul_rn(__fadd_rn(a[i], s[i]), inv_n);
    a[i] = 0.f;
  }
}

extern "C" {

void atomo_v2_launch_accum_add(const void* wchunks, int nw, const void* vchunks, int nv, const long long* gptr,
                               float* acc, float* vacc, float* vgrads, int first, cudaStream_t stream) {
  if (nw + nv <= 0) return;
  v2_accum_add_kernel<<<nw + nv, ACC_THREADS, 0, stream>>>((const EfChunk*)wchunks, nw, (const EfChunk*)vchunks,
                                                           gptr, acc, vacc, vgrads, first);
}

void atomo_v2_launch_accum_fold(const void* wchunks, int nw, const void* vchunks, int nv, const long long* gptr,
                                float* acc, float* vacc, float* vgrads, float inv_n, float* residual,
                                cudaStream_t stream) {
  if (nw + nv <= 0) return;
  v2_accum_fold_kernel<<<nw + nv, ACC_THREADS, 0, stream>>>((const EfChunk*)wchunks, nw, (const EfChunk*)vchunks,
                                                            gptr, acc, vacc, vgrads, inv_n, residual);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
