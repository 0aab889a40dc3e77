// Exponential moving average of the weights on the overlapped, sharded bf16 engine (sm_90a): one backward group of one
// owner (ShadowEngine(ema_decay=d)).
//
// On the PS stream, right after the launch that writes the group's final master values (the PS launch, LARS / LAMB
// phase 2 or the clip launch), this launch walks the owner's PS tiles of the group, the contiguous range the PS took,
// and averages every fp32 value the owner holds:
//
//   e <- e + w (p - e),   w = fp32(1 - d) from the host
//
// p the value after the step: a weight tile's elements of master (lw_tile_segs) into ema, a vector tile's elements of
// vparams into vema.  Each operation is a named round-to-nearest intrinsic, so a numpy float32 oracle matches the pass
// bit for bit.  Bandwidth bound: p and e read, e written, 12 bytes per element.  vparams is read with ld.global.cg:
// the PS stored it through multicast or peer stores.
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int EMA_THREADS = 256;

__device__ __forceinline__ float ema_step(float e, float p, float w) {
  return __fadd_rn(e, __fmul_rn(w, __fsub_rn(p, e)));
}

// the tiles of the launch are split into contiguous runs per CTA, as the PS kernels split them (ps_tile_range)
__global__ void __launch_bounds__(EMA_THREADS) v2_ema_kernel(const Unit2* units, const Tile2* tiles, int ntiles,
                                                              const float* master, const float* vparams, float* ema,
                                                              float* vema, float w) {
  const int per_cta = (ntiles + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta, t_end = min(ntiles, t_begin + per_cta);
  for (int ti = t_begin; ti < t_end; ++ti) {
    const Tile2 t = tiles[ti];
    const Unit2& u = units[t.unit];
    const bool is_vec = u.kind == KIND_VEC;
    LwSegs sg;
    if (is_vec) {
      sg.nseg = 1; sg.seglen = t.b; sg.segbase = u.w_off + t.a; sg.segstride = 0;
    } else {
      sg = lw_tile_segs(u, t);
    }
    const float* p = (is_vec ? vparams : master) + sg.segbase;
    float* e = (is_vec ? vema : ema) + sg.segbase;
    // float4 over each segment when its start and stride are 16-byte aligned; the segment's last seglen % 4 elements
    // (or all of them otherwise) take the scalar loop
    const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(e)) & 15) == 0 &&
                     (sg.segstride & 3) == 0;
    const int spv = vec ? (sg.seglen >> 2) : 0, tail = sg.seglen - 4 * spv;
    for (int v = threadIdx.x; v < sg.nseg * spv; v += EMA_THREADS) {
      const int s = v / spv, i4 = v - s * spv;
      const long long o = s * sg.segstride + 4LL * i4;
      const float4 x = ld_cg_f4(reinterpret_cast<const float4*>(p + o));
      float4 y = *reinterpret_cast<const float4*>(e + o);
      y.x = ema_step(y.x, x.x, w);
      y.y = ema_step(y.y, x.y, w);
      y.z = ema_step(y.z, x.z, w);
      y.w = ema_step(y.w, x.w, w);
      *reinterpret_cast<float4*>(e + o) = y;
    }
    for (int v = threadIdx.x; v < sg.nseg * tail; v += EMA_THREADS) {
      const int s = v / tail, i = v - s * tail;
      const long long o = s * sg.segstride + 4LL * spv + i;
      e[o] = ema_step(e[o], ld_cg_f(p + o), w);
    }
  }
}

extern "C" {

void atomo_v2_launch_ema(const void* units, const void* tiles, int tile0, int ntiles, const float* master,
                         const float* vparams, float* ema, float* vema, float w, int grid, cudaStream_t stream) {
  if (ntiles <= 0) return;
  v2_ema_kernel<<<ps_grid(grid, ntiles), EMA_THREADS, 0, stream>>>((const Unit2*)units, (const Tile2*)tiles + tile0,
                                                                    ntiles, master, vparams, ema, vema, w);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
