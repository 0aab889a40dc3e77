// Error feedback on the overlapped, sharded bf16 engine (sm_90a): the apply pass of ONE backward group.
//
// Each worker keeps an fp32 residual e per weight element, in the physical order of wshadow, and codes A = g + e
// instead of its gradient g.  The residual is formed in two places:
//
//   v2_ef_apply_kernel   before the group's encode, on the encode stream: A = g + e in fp32, bf16(A) written back in
//                        place into autograd's gradient buffer (through the pointer table, so the encoders code A
//                        without any change to how they read it), and the rounding remainder A - bf16(A) stored into
//                        the residual.  Bandwidth bound: 2 + 4 bytes read and 2 + 4 bytes written per element, with
//                        16-byte loads and stores.
//   encoder epilogues    v2_entry_encode_kernel, v2_qsgd_encode_kernel and v2_project_kernel add bf16(A) - g_hat to
//                        the residual, with g_hat the values this worker pushed (a null residual pointer: no epilogue).
//
// After both, e = A - g_hat: nothing the code drops is lost, it is sent in a later step.
#include "v2_common.cuh"

namespace atomo {
namespace v2 {

constexpr int EF_THREADS = 256;

// One apply chunk: `count` consecutive elements of weight tensor `widx` from element `start`; the tensor's first
// element is residual element `w_off` (ops/plan2.py: Plan2.ef_chunks, the layout is mirrored there)
struct EfChunk {
  long long w_off;
  int widx;
  int start;
  int count;
  int pad;
};
static_assert(sizeof(EfChunk) == 24, "EfChunk layout must match ops/plan2.py EF_CHUNK_FMT");

__device__ __forceinline__ float ef_round(float a, __nv_bfloat16& b) {
  b = __float2bfloat16_rn(a);
  return a - __bfloat162float(b);      // exact: the part of a that bf16 cannot hold
}

__global__ void __launch_bounds__(EF_THREADS) v2_ef_apply_kernel(const EfChunk* chunks, const long long* gptr,
                                                                  float* residual) {
  const EfChunk c = chunks[blockIdx.x];
  __nv_bfloat16* g = reinterpret_cast<__nv_bfloat16*>(gptr[c.widx]) + c.start;
  float* e = residual + c.w_off + c.start;
  // 8 elements per 16-byte bf16 access (two 16-byte residual accesses); chunks start on multiples of 8 elements, so
  // only a gradient buffer that autograd hands over unaligned takes the scalar path
  const bool vec = ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(e)) & 15) == 0;
  const int nv = vec ? (c.count >> 3) : 0;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    uint4 gw = *reinterpret_cast<const uint4*>(g + 8 * v);
    float4 e0 = reinterpret_cast<const float4*>(e)[2 * v];
    float4 e1 = reinterpret_cast<const float4*>(e)[2 * v + 1];
    const float x[8] = {bf16_lo(gw.x), bf16_hi(gw.x), bf16_lo(gw.y), bf16_hi(gw.y),
                        bf16_lo(gw.z), bf16_hi(gw.z), bf16_lo(gw.w), bf16_hi(gw.w)};
    float r[8] = {e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w};
    __nv_bfloat16 b[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = ef_round(__fadd_rn(x[i], r[i]), b[i]);
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      w[i] = (uint32_t)__bfloat16_as_ushort(b[2 * i]) | ((uint32_t)__bfloat16_as_ushort(b[2 * i + 1]) << 16);
    gw = make_uint4(w[0], w[1], w[2], w[3]);
    *reinterpret_cast<uint4*>(g + 8 * v) = gw;
    reinterpret_cast<float4*>(e)[2 * v] = make_float4(r[0], r[1], r[2], r[3]);
    reinterpret_cast<float4*>(e)[2 * v + 1] = make_float4(r[4], r[5], r[6], r[7]);
  }
  for (int i = (nv << 3) + threadIdx.x; i < c.count; i += blockDim.x) {
    __nv_bfloat16 b;
    e[i] = ef_round(__fadd_rn(__bfloat162float(g[i]), e[i]), b);
    g[i] = b;
  }
}

extern "C" {

int atomo_v2_ef_chunk_bytes() { return (int)sizeof(EfChunk); }

void atomo_v2_launch_ef_apply(const void* chunks, int chunk0, int nchunks, const long long* gptr, float* residual,
                              cudaStream_t stream) {
  if (nchunks <= 0) return;
  v2_ef_apply_kernel<<<nchunks, EF_THREADS, 0, stream>>>((const EfChunk*)chunks + chunk0, gptr, residual);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
