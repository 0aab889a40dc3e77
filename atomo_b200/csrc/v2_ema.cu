// Owner-local passes over one backward group's PS tiles on the overlapped, sharded bf16 engine (sm_90a): the
// exponential moving average of the weights (ShadowEngine(ema_decay=d)) and the decoupled weight decay of AdamW
// (ShadowEngine(optimizer="adamw")).  Both walk the owner's PS tiles of the group, the contiguous range the PS takes,
// with the same grid and the same segments (owner_tile_walk below); only the per-element step differs.
//
// Average: on the PS stream, right after the launch that writes the group's final master values (the PS launch, LARS /
// LAMB phase 2 or the clip launch), every fp32 value the owner holds is averaged:
//
//   e <- e + w (p - e),   w = fp32(1 - d) from the host
//
// p the value after the step: a weight tile's elements of master (lw_tile_segs) into ema, a vector tile's elements of
// vparams into vema.  Each operation is a named round-to-nearest intrinsic, so a numpy float32 oracle matches the pass
// bit for bit.  Bandwidth bound: p and e read, e written, 12 bytes per element.  vparams is read with ld.global.cg:
// the PS stored it through multicast or peer stores.
//
// Decoupled weight decay: on the PS stream, right before the launch that steps the group's tiles (the PS launch, or
// with clipping the clip launch), every weight element of master the owner holds is scaled:
//
//   p <- p * f,   f = Ctrl2::decay_factor = fp32(1 - lr wd), rewritten by the host with every set_lr
//
// one __fmul_rn per element, so torch's fp32 p.mul_(f) matches bit for bit.  Vector tiles (BN, biases) are skipped:
// AdamW's second parameter group takes no decay.  f is read from Ctrl2, never from an argument, so a captured graph
// sees every LR change.  Only owner-local master is written, which no forward or backward reads (the workers read the
// bf16 broadcast the PS writes after the step), so the pass needs no wait of its own.  8 bytes per weight element.
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int EMA_THREADS = 256;

__device__ __forceinline__ float ema_step(float e, float p, float w) {
  return __fadd_rn(e, __fmul_rn(w, __fsub_rn(p, e)));
}

// The tiles of the launch are split into contiguous runs per CTA, as the PS kernels split them (ps_tile_range).  Each
// tile is a set of equal segments of its source p and destination e: a weight tile's elements (lw_tile_segs) of wsrc
// and wdst, a vector tile's of vsrc and vdst.  Every element becomes e = step(e, p); without kSource p is not read
// (step gets 0), and without kVectors vector tiles are skipped.
template <bool kVectors, bool kSource, class Step>
__device__ __forceinline__ void owner_tile_walk(const Unit2* units, const Tile2* tiles, int ntiles, const float* wsrc,
                                                const float* vsrc, float* wdst, float* vdst, Step step) {
  const int per_cta = (ntiles + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta, t_end = min(ntiles, t_begin + per_cta);
  for (int ti = t_begin; ti < t_end; ++ti) {
    const Tile2 t = tiles[ti];
    const Unit2& u = units[t.unit];
    const bool is_vec = u.kind == KIND_VEC;
    if (!kVectors && is_vec) continue;
    LwSegs sg;
    if (is_vec) {
      sg.nseg = 1; sg.seglen = t.b; sg.segbase = u.w_off + t.a; sg.segstride = 0;
    } else {
      sg = lw_tile_segs(u, t);
    }
    const float* p = (is_vec ? vsrc : wsrc) + sg.segbase;
    float* e = (is_vec ? vdst : wdst) + sg.segbase;
    // float4 over each segment when its start and stride are 16-byte aligned; the segment's last seglen % 4 elements
    // (or all of them otherwise) take the scalar loop
    const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(e)) & 15) == 0 &&
                     (sg.segstride & 3) == 0;
    const int spv = vec ? (sg.seglen >> 2) : 0, tail = sg.seglen - 4 * spv;
    for (int v = threadIdx.x; v < sg.nseg * spv; v += EMA_THREADS) {
      const int s = v / spv, i4 = v - s * spv;
      const long long o = s * sg.segstride + 4LL * i4;
      const float4 x = kSource ? ld_cg_f4(reinterpret_cast<const float4*>(p + o)) : float4{};
      float4 y = *reinterpret_cast<const float4*>(e + o);
      y.x = step(y.x, x.x);
      y.y = step(y.y, x.y);
      y.z = step(y.z, x.z);
      y.w = step(y.w, x.w);
      *reinterpret_cast<float4*>(e + o) = y;
    }
    for (int v = threadIdx.x; v < sg.nseg * tail; v += EMA_THREADS) {
      const int s = v / tail, i = v - s * tail;
      const long long o = s * sg.segstride + 4LL * spv + i;
      e[o] = step(e[o], kSource ? ld_cg_f(p + o) : 0.f);
    }
  }
}

struct EmaStep {
  float w;
  __device__ __forceinline__ float operator()(float e, float p) const { return ema_step(e, p, w); }
};

// in place on master, weight tiles only: p is not read
struct DecayStep {
  float f;
  __device__ __forceinline__ float operator()(float e, float) const { return __fmul_rn(e, f); }
};

__global__ void __launch_bounds__(EMA_THREADS) v2_ema_kernel(const Unit2* units, const Tile2* tiles, int ntiles,
                                                              const float* master, const float* vparams, float* ema,
                                                              float* vema, float w) {
  owner_tile_walk<true, true>(units, tiles, ntiles, master, vparams, ema, vema, EmaStep{w});
}

__global__ void __launch_bounds__(EMA_THREADS) v2_decay_kernel(const Unit2* units, const Tile2* tiles, int ntiles,
                                                                float* master, const Ctrl2* ctrl) {
  owner_tile_walk<false, false>(units, tiles, ntiles, master, master, master, master, DecayStep{ctrl->decay_factor});
}

extern "C" {

void atomo_v2_launch_ema(const void* units, const void* tiles, int tile0, int ntiles, const float* master,
                         const float* vparams, float* ema, float* vema, float w, int grid, cudaStream_t stream) {
  if (ntiles <= 0) return;
  v2_ema_kernel<<<ps_grid(grid, ntiles), EMA_THREADS, 0, stream>>>((const Unit2*)units, (const Tile2*)tiles + tile0,
                                                                    ntiles, master, vparams, ema, vema, w);
}

void atomo_v2_launch_decay(const void* units, const void* tiles, int tile0, int ntiles, float* master,
                           const void* ctrl, int grid, cudaStream_t stream) {
  if (ntiles <= 0) return;
  v2_decay_kernel<<<ps_grid(grid, ntiles), EMA_THREADS, 0, stream>>>((const Unit2*)units, (const Tile2*)tiles + tile0,
                                                                      ntiles, master, (const Ctrl2*)ctrl);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
