// Parameter-server building blocks shared by the PS kernels of the overlapped / sharded engine: the launch
// arguments, the push wait with the --num-aggregate mask and the prologue around it, the stale-slot check, the fp32
// vector and dense bf16 tiles, the fused optimizer epilogue with its bf16 broadcast, the completion, and the host
// packing of the launch arguments.  Every v2_ps*_kernel uses them (v2_ps.cu, v2_qsgd.cu, v2_entrywise.cu, v2_sign.cu,
// v2_fp8.cu, v2_hadamard.cu, v2_powersgd.cu); v2_ps_kernel keeps its own copies where noted.
#pragma once
#include <type_traits>

#include "v2_common.cuh"
#include "v2_momentum.cuh"

namespace atomo {
namespace v2 {

struct PsArgs2 {
  const Unit2* units;
  const Tile2* tiles;
  int ntiles;
  int W;
  int nranks;
  int group;
  int final_group;
  int owner;
  float* master; float* mom; float* sq; float* sqmax;       // indexed like wshadow (owner-local fp32 state)
  float* vmom; float* vsq; float* vsqmax;                   // indexed like vparams
  __nv_bfloat16* wshadow_mc; __nv_bfloat16* const* wshadow_peer;
  float* vparams_local; float* vparams_mc; float* const* vparams_peer;
  const float* vgrads_mc; const float* const* vgrads_peer;  // [W]
  const __nv_bfloat16* const* stage_peer;                   // [W]
  const float* arenas;
  long long arena_floats;
  int* sig;
  int* const* sig_peer;
  Ctrl2* ctrl;
  unsigned int* group_counter;
  long long timeout;
  long long* tstats;
  float inv_w;
};

struct OptC {
  float lr, mu, damp, wd, b1, b2, eps, bc1, sbc2;
  int nesterov, first, opt;
};

__device__ __forceinline__ void opt_update(float g, float& p, float& m, float& v, float& vmax, const OptC& c) {
  g = fmaf(c.wd, p, g);
  if (c.opt == OPT_SGD) {
    float d = g;
    if (c.mu != 0.f) {
      m = c.first ? g : fmaf(c.mu, m, (1.f - c.damp) * g);
      d = c.nesterov ? fmaf(c.mu, m, g) : m;
    }
    p = fmaf(-c.lr, d, p);
  } else {
    m = fmaf(c.b1, m, (1.f - c.b1) * g);
    v = fmaf(c.b2, v, (1.f - c.b2) * g * g);
    float vv = v;
    if (c.opt == OPT_AMSGRAD) { vmax = fmaxf(vmax, v); vv = vmax; }
    const float denom = sqrtf(vv) / c.sbc2 + c.eps;
    p -= (c.lr / c.bc1) * (m / denom);
  }
}

// ---- layer-wise optimizers (LARS / LAMB), phase 1 -----------------------------------------------------------------
// A trust ratio needs whole-tensor norms before any element of the tensor moves, and no owner sees a whole tensor.
// So every PS kernel has a layer-wise instantiation (its body is a template over the argument type): where the plain one
// steps the optimizer and broadcasts, it writes the direction x (LARS: d = g + wd w; LAMB: u, after the Adam moments)
// to `dir` and adds (w^2, x^2) to the thread's partial; the partials are reduced in a fixed order per PS tile into
// `part`.  Weights are neither written nor broadcast: v2_layerwise.cu (phase 2) takes the norms across tiles and owners
// and steps them.  Vector tiles are finished here: momentum-SGD (LARS) or Adam (LAMB), without weight decay.
constexpr int LW_THREADS = 256;   // every PS kernel runs 256 threads

struct PsArgsLw : PsArgs2 {
  float* dir;      // direction, indexed like master (owner-local scratch)
  float2* part;    // per PS tile of the launch: (sum w^2, sum x^2)
};

template <class A>
constexpr bool ps_layerwise = std::is_same<A, PsArgsLw>::value;

// ---- gradient-norm clipping, phase 1 ("gather") ------------------------------------------------------------------
// The clip coefficient needs the norm of the whole step's gradient, summed over every group and owner, before any
// element moves.  So with clipping on, every PS kernel runs its gather instantiation: it stores the mean gradient g
// (the value the plain instantiation hands to the optimizer) into owner-local fp32 scratch and reduces sum g^2 per PS
// tile, vector tiles included, in a fixed order into part[ti].x.  It steps, broadcasts and publishes nothing:
// v2_clip.cu (phase 2) takes the norm across tiles and owners and steps every tile of the owner.
struct PsArgsGather : PsArgs2 {
  float* grad;     // g, indexed like master (owner-local scratch)
  float* vgrad;    // g of the vector tiles, indexed like vparams
  float2* part;    // per PS tile of the launch: (sum g^2, 0)
};

template <class A>
constexpr bool ps_gather = std::is_same<A, PsArgsGather>::value;

// the instantiations that reduce a partial per PS tile into a.part (lw_begin / lw_tile_done)
template <class A>
constexpr bool ps_tile_partials = ps_layerwise<A> || ps_gather<A>;

__shared__ float2 lw_acc[LW_THREADS];    // one partial per thread, reduced and zeroed at the end of every weight tile

// the direction of one weight element and its partials (lw_acc of this thread)
__device__ __forceinline__ float lw_direction(const PsArgsLw& a, const OptC& c, long long e, float g, float p,
                                              float2& acc) {
  float x;
  if (c.opt == OPT_LARS) {
    x = fmaf(c.wd, p, g);
    acc.y = fmaf(g, g, acc.y);
  } else {
    float m = a.mom[e], v = a.sq[e];
    m = fmaf(c.b1, m, (1.f - c.b1) * g);
    v = fmaf(c.b2, v, (1.f - c.b2) * g * g);
    a.mom[e] = m;
    a.sq[e] = v;
    x = fmaf(c.wd, p, (m / c.bc1) / (sqrtf(v) / c.sbc2 + c.eps));
    acc.y = fmaf(x, x, acc.y);
  }
  acc.x = fmaf(p, p, acc.x);
  return x;
}

__device__ __forceinline__ void update8(const PsArgsLw& a, const OptC& c, long long e, const float (&g)[8]) {
  float2 acc = lw_acc[threadIdx.x];
  const float4 p0 = *reinterpret_cast<const float4*>(a.master + e), p1 = *reinterpret_cast<const float4*>(a.master + e + 4);
  const float p[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
  float x[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = lw_direction(a, c, e + i, g[i], p[i], acc);
  *reinterpret_cast<float4*>(a.dir + e) = make_float4(x[0], x[1], x[2], x[3]);
  *reinterpret_cast<float4*>(a.dir + e + 4) = make_float4(x[4], x[5], x[6], x[7]);
  lw_acc[threadIdx.x] = acc;
}

__device__ __forceinline__ void update1(const PsArgsLw& a, const OptC& c, long long e, float g) {
  float2 acc = lw_acc[threadIdx.x];
  a.dir[e] = lw_direction(a, c, e, g, a.master[e], acc);
  lw_acc[threadIdx.x] = acc;
}

__device__ __forceinline__ void update8(const PsArgsGather& a, const OptC&, long long e, const float (&g)[8]) {
  float2 acc = lw_acc[threadIdx.x];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc.x = fmaf(g[i], g[i], acc.x);
  *reinterpret_cast<float4*>(a.grad + e) = make_float4(g[0], g[1], g[2], g[3]);
  *reinterpret_cast<float4*>(a.grad + e + 4) = make_float4(g[4], g[5], g[6], g[7]);
  lw_acc[threadIdx.x] = acc;
}

__device__ __forceinline__ void update1(const PsArgsGather& a, const OptC&, long long e, float g) {
  lw_acc[threadIdx.x].x = fmaf(g, g, lw_acc[threadIdx.x].x);
  a.grad[e] = g;
}

// start of the launch: zero partials
template <class A>
__device__ __forceinline__ void lw_begin(const A&) {
  if constexpr (ps_tile_partials<A>) lw_acc[threadIdx.x] = make_float2(0.f, 0.f);
}

// end of PS tile ti (every thread of the CTA): the partials summed in a fixed order into part[ti], then zeroed
template <class A>
__device__ __forceinline__ void lw_tile_done(const A& a, int ti) {
  if constexpr (ps_tile_partials<A>) {
    __shared__ float2 wsum[LW_THREADS / 32];
    float2 v = lw_acc[threadIdx.x];
    lw_acc[threadIdx.x] = make_float2(0.f, 0.f);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
      v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    }
    __syncthreads();   // every lane's epilogue is done, and the previous tile's wsum has been read
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
      float2 s = wsum[0];
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { s.x += wsum[w].x; s.y += wsum[w].y; }
      a.part[ti] = s;
    }
  }
}

// The elements of PS tile t of unit u: nseg segments of seglen elements, segstride apart, from segbase (the tiles of
// v2_ps_kernel's low-rank epilogue, of PowerSGD's row tiles, and of every code whose tiles are consecutive elements)
struct LwSegs {
  int nseg, seglen;
  long long segbase, segstride;
};

__device__ __forceinline__ LwSegs lw_tile_segs(const Unit2& u, const Tile2& t) {
  LwSegs s;
  if (u.kind == KIND_SLAB) {
    const int half = u.I >> 1;
    s.nseg = 1; s.seglen = (t.b / half) * u.K * u.I; s.segbase = u.w_off + (long long)(t.a / half) * u.K * u.I;
    s.segstride = 0;
  } else if (u.kind == KIND_MAT && u.cs == 1) {
    s.nseg = t.b; s.seglen = u.cols; s.segbase = u.w_off + (long long)t.a * u.rs; s.segstride = u.rs;
  } else if (u.kind == KIND_MAT) {
    s.nseg = u.cols; s.seglen = t.b; s.segbase = u.w_off + t.a; s.segstride = u.cs;
  } else if (u.kind == KIND_POWER) {
    s.nseg = 1; s.seglen = t.b * u.cols; s.segbase = u.w_off + (long long)t.a * u.cols; s.segstride = 0;
  } else {
    s.nseg = 1; s.seglen = t.b; s.segbase = u.w_off + t.a; s.segstride = 0;
  }
  return s;
}

__device__ __forceinline__ uint4 ld_cg_u4(const void* p) {
  uint4 v;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_cg_bf16(const __nv_bfloat16* p) {
  unsigned short h;
  asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(h) : "l"(p));
  return __uint_as_float((uint32_t)h << 16);
}

__device__ __forceinline__ uint4 pack_bf16x8(const float (&f)[8]) {
  uint4 r;
  __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return r;
}

__device__ __forceinline__ void mc_store16(void* mc, const uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
               : "memory");
}

// the bf16 copy of 8 consecutive updated weights from element e (16-byte aligned in bf16) to every rank
__device__ __forceinline__ void ps_bcast8(const PsArgs2& a, long long e, const float (&p)[8]) {
  const uint4 packed = pack_bf16x8(p);
  if (a.wshadow_mc != nullptr) {
    mc_store16(a.wshadow_mc + e, packed);
  } else {
    for (int r = 0; r < a.nranks; ++r) *reinterpret_cast<uint4*>(a.wshadow_peer[r] + e) = packed;
  }
}

// ... of one updated weight (the scalar tail: peer stores only)
__device__ __forceinline__ void ps_bcast1(const PsArgs2& a, long long e, float p) {
  const __nv_bfloat16 b = __float2bfloat16_rn(p);
  for (int r = 0; r < a.nranks; ++r) a.wshadow_peer[r][e] = b;
}

// update 8 consecutive weight elements starting at element e (16-byte aligned in bf16), broadcast the bf16 copy
__device__ __forceinline__ void update8(const PsArgs2& a, const OptC& c, long long e, const float (&g)[8]) {
  float p[8], m[8], v[8], vm[8];
  const float4 p0 = *reinterpret_cast<const float4*>(a.master + e), p1 = *reinterpret_cast<const float4*>(a.master + e + 4);
  const float4 m0 = *reinterpret_cast<const float4*>(a.mom + e), m1 = *reinterpret_cast<const float4*>(a.mom + e + 4);
  p[0] = p0.x; p[1] = p0.y; p[2] = p0.z; p[3] = p0.w; p[4] = p1.x; p[5] = p1.y; p[6] = p1.z; p[7] = p1.w;
  m[0] = m0.x; m[1] = m0.y; m[2] = m0.z; m[3] = m0.w; m[4] = m1.x; m[5] = m1.y; m[6] = m1.z; m[7] = m1.w;
  if (c.opt != OPT_SGD) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i] = a.sq[e + i]; vm[i] = c.opt == OPT_AMSGRAD ? a.sqmax[e + i] : 0.f; }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i] = 0.f; vm[i] = 0.f; }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) opt_update(g[i], p[i], m[i], v[i], vm[i], c);
  *reinterpret_cast<float4*>(a.master + e) = make_float4(p[0], p[1], p[2], p[3]);
  *reinterpret_cast<float4*>(a.master + e + 4) = make_float4(p[4], p[5], p[6], p[7]);
  *reinterpret_cast<float4*>(a.mom + e) = make_float4(m[0], m[1], m[2], m[3]);
  *reinterpret_cast<float4*>(a.mom + e + 4) = make_float4(m[4], m[5], m[6], m[7]);
  if (c.opt != OPT_SGD) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { a.sq[e + i] = v[i]; if (c.opt == OPT_AMSGRAD) a.sqmax[e + i] = vm[i]; }
  }
  ps_bcast8(a, e, p);
}

__device__ __forceinline__ void update1(const PsArgs2& a, const OptC& c, long long e, float g) {
  float p = a.master[e], m = a.mom[e], v = 0.f, vm = 0.f;
  if (c.opt != OPT_SGD) { v = a.sq[e]; if (c.opt == OPT_AMSGRAD) vm = a.sqmax[e]; }
  opt_update(g, p, m, v, vm, c);
  a.master[e] = p; a.mom[e] = m;
  if (c.opt != OPT_SGD) { a.sq[e] = v; if (c.opt == OPT_AMSGRAD) a.sqmax[e] = vm; }
  ps_bcast1(a, e, p);
}

// ---- Lion (Chen et al. 2023), the fourth instantiation of every PS kernel -----------------------------------------
// Per element, on the mean gradient g the plain instantiation hands to the optimizer, every operation rounded on its
// own (no contraction), om1 = 1 - b1 and om2 = 1 - b2 formed in fp32:
//   c = b1 m + om1 g;  p <- p - lr sign(c);  m <- b2 m + om2 g
// sign(+-0) = 0, so an exact zero c leaves p as it was; a NaN c gives a NaN step (torch.sign would return 0 and hide
// it).  m starts at zero; no bias correction.  The decoupled weight decay of the weights is the v2_decay launch before
// this one (Ctrl2::decay_factor).  State: master and mom (vectors: vparams and vmom); sq / sqmax / vsq / vsqmax are
// never touched.  Then the same bf16 (weights) or fp32 (vectors) broadcast as the plain instantiation.
struct PsArgsLion : PsArgs2 {};

__device__ __forceinline__ void lion_update(float g, float& p, float& m, const OptC& c) {
  const float cc = lion_direction(g, m, c.b1);      // v2_momentum.cuh: Distributed Lion's workers round the same way
  const float s = cc > 0.f ? 1.f : cc < 0.f ? -1.f : cc == 0.f ? 0.f : cc;
  p = __fsub_rn(p, __fmul_rn(c.lr, s));
  m = lion_momentum(g, m, c.b2);
}

__device__ __forceinline__ void update8(const PsArgsLion& a, const OptC& c, long long e, const float (&g)[8]) {
  const float4 p0 = *reinterpret_cast<const float4*>(a.master + e), p1 = *reinterpret_cast<const float4*>(a.master + e + 4);
  const float4 m0 = *reinterpret_cast<const float4*>(a.mom + e), m1 = *reinterpret_cast<const float4*>(a.mom + e + 4);
  float p[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
  float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
#pragma unroll
  for (int i = 0; i < 8; ++i) lion_update(g[i], p[i], m[i], c);
  *reinterpret_cast<float4*>(a.master + e) = make_float4(p[0], p[1], p[2], p[3]);
  *reinterpret_cast<float4*>(a.master + e + 4) = make_float4(p[4], p[5], p[6], p[7]);
  *reinterpret_cast<float4*>(a.mom + e) = make_float4(m[0], m[1], m[2], m[3]);
  *reinterpret_cast<float4*>(a.mom + e + 4) = make_float4(m[4], m[5], m[6], m[7]);
  ps_bcast8(a, e, p);
}

__device__ __forceinline__ void update1(const PsArgsLion& a, const OptC& c, long long e, float g) {
  float p = a.master[e], m = a.mom[e];
  lion_update(g, p, m, c);
  a.master[e] = p; a.mom[e] = m;
  ps_bcast1(a, e, p);
}

// ---- push wait (thread 0 of every CTA) ------------------------------------------------------------------
// Default: all W workers.  With Ctrl2::num_aggregate = N < W (the reference's --num-aggregate, parsed at
// distributed_nn.py:67 and never used there) the owner proceeds as soon as N pushes of THIS step have landed:
// CTA 0 decides the set once and publishes it (mask, then a step stamp) so that every CTA of the launch
// averages the same workers; late pushes carry an older step in their flag and are simply never counted.
// Returns false on a timeout; `mask` receives the set of workers to average.
// v2_ps_kernel keeps its own inline copy of this wait and of ps_opt_consts: calling these functions there
// changes its register allocation and instruction schedule.  Keep the two copies in step.
__device__ __forceinline__ bool ps_wait_pushes(const PsArgs2& a, const Ctrl2* ctrl, int step, unsigned int& mask) {
  bool ok = true;
  const int* flags = a.sig + SIG_PUSH + a.group * MAX_WORKERS;
  const int need = (ctrl->num_aggregate > 0 && ctrl->num_aggregate < a.W) ? ctrl->num_aggregate : a.W;
  mask = a.W >= 32 ? 0xffffffffu : ((1u << a.W) - 1u);
  if (need == a.W) {
    for (int w = 0; w < a.W; ++w) ok = spin_wait_ge(flags + w, step, a.timeout) && ok;
  } else {
    int* mslot = a.sig + SIG_MASK + 2 * a.group;
    if (blockIdx.x == 0) {
      const long long t0 = clock64();
      int backoff = 32;
      for (;;) {
        mask = 0;
        int n = 0;
        for (int w = 0; w < a.W; ++w)
          if (ld_acquire_sys(flags + w) >= step) { mask |= 1u << w; ++n; }
        if (n >= need) break;
        __nanosleep(backoff);
        if (backoff < 1024) backoff <<= 1;
        if (clock64() - t0 > a.timeout) { ok = false; break; }
      }
      mslot[0] = (int)mask;
      __threadfence();
      asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(mslot + 1), "r"(ok ? step : -step) : "memory");
    } else {
      int v;
      const long long t0 = clock64();
      do {
        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(mslot + 1) : "memory");
        if (clock64() - t0 > 2 * a.timeout) { v = -step; break; }
      } while (v != step && v != -step);
      ok = v == step;
      mask = (unsigned int)ld_cg_i(mslot);
    }
  }
  return ok;
}

// ---- PS prologue: thread 0 waits for the pushes, then every thread reads the outcome -----------------------------
// ok / bad / mask are the CTA's shared flags; t_enter / t_ready are thread 0's timings (shared or registers).
__device__ __forceinline__ void ps_wait(const PsArgs2& a, Ctrl2* ctrl, int step, int& s_ok, int& s_bad,
                                        unsigned int& s_mask, long long& t_enter, long long& t_ready) {
  if (threadIdx.x == 0) {
    t_enter = globaltimer_ns();
    unsigned int mask;
    const bool ok = ps_wait_pushes(a, ctrl, step, mask);
    if (!ok) atomicOr(&ctrl->error, ERR2_WAIT_PUSH);
    s_ok = ok ? 1 : 0;
    s_bad = 0;
    s_mask = mask;
    t_ready = globaltimer_ns();
  }
  __syncthreads();
}

// The CTA's range of tiles [t_begin, t_end): consecutive tiles, the same count per CTA but for the last.
struct PsTiles {
  int t_begin, t_end;
};

__device__ __forceinline__ PsTiles ps_tile_range(const PsArgs2& a) {
  const int per_cta = (a.ntiles + gridDim.x - 1) / gridDim.x;
  PsTiles r;
  r.t_begin = blockIdx.x * per_cta;
  r.t_end = min(a.ntiles, r.t_begin + per_cta);
  return r;
}

// ---- stale-slot check (thread 0, per tile): the counted workers whose stamp for the tile, stamp_of(w), is this
// step; any other stamp is a push of another step and sets `bad` (ERR2_SLOT_STEP in ps_complete).
template <class StampOf>
__device__ __forceinline__ unsigned int ps_fresh_workers(const PsArgs2& a, unsigned int wmask, int step, int& bad,
                                                         StampOf stamp_of) {
  unsigned int use = 0;
  for (int w = 0; w < a.W; ++w) {
    if (!((wmask >> w) & 1u)) continue;
    if (ld_cg_i(stamp_of(w)) == step) use |= 1u << w;
    else bad = 1;
  }
  return use;
}

// ... for the slots that start with one int32 stamp per PS tile (QSGD, sign, fp8, hadamard, powersgd): stamp jt
__device__ __forceinline__ unsigned int ps_fresh_workers(const PsArgs2& a, const Unit2& u, int jt, unsigned int wmask,
                                                         int step, int& bad) {
  return ps_fresh_workers(a, wmask, step, bad, [&](int w) {
    return reinterpret_cast<const int*>(a.arenas + (long long)w * a.arena_floats + u.slot_off) + jt;
  });
}

__device__ __forceinline__ OptC ps_opt_consts(const Ctrl2* ctrl, int step) {
  OptC c;
  c.lr = ctrl->lr; c.mu = ctrl->momentum; c.damp = ctrl->dampening; c.wd = ctrl->weight_decay;
  c.nesterov = ctrl->nesterov; c.first = (step == ctrl->first_step); c.opt = ctrl->opt;
  c.b1 = ctrl->beta1; c.b2 = ctrl->beta2; c.eps = ctrl->eps;
  {
    const float t = (float)(step - ctrl->first_step + 1);
    c.bc1 = 1.f - powf(c.b1, t);
    c.sbc2 = sqrtf(1.f - powf(c.b2, t));
  }
  return c;
}

// ---- fp32 vector tile (BN, biases): sum of the counted workers' gradients, optimizer, fp32 broadcast ------------
// The walk is shared by the plain and the Lion instantiation: step4(e, g, p) / step1(e, g, p) update the vector
// element(s) at e in p (read from vparams_local) from the workers' gradient sum g and write their own state.
template <class Step4, class Step1>
__device__ __forceinline__ void ps_vec_walk(const PsArgs2& a, const Unit2& u, const Tile2& t, unsigned int wmask,
                                            bool all_workers, Step4 step4, Step1 step1) {
  const int tid = threadIdx.x;
  const long long e0 = u.w_off + t.a;
  const int nvec = t.b >> 2;
  for (int v = tid; v < nvec; v += blockDim.x) {
    const long long e = e0 + 4LL * v;
    float4 g;
    if (a.vgrads_mc != nullptr && all_workers) {
      g = multimem_ld_reduce_f4(reinterpret_cast<const float4*>(a.vgrads_mc + e));
    } else {
      g = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int w = 0; w < a.W; ++w) {
        if (!((wmask >> w) & 1u)) continue;
        const float4 x = ld_cg_f4(reinterpret_cast<const float4*>(a.vgrads_peer[w] + e));
        g.x += x.x; g.y += x.y; g.z += x.z; g.w += x.w;
      }
    }
    float4 p = *reinterpret_cast<float4*>(a.vparams_local + e);
    step4(e, g, p);
    if (a.vparams_mc != nullptr) {
      multimem_st_f4(reinterpret_cast<float4*>(a.vparams_mc + e), p);
    } else {
      for (int r = 0; r < a.nranks; ++r) st_na_f4(reinterpret_cast<float4*>(a.vparams_peer[r] + e), p);
    }
  }
  for (int i = (nvec << 2) + tid; i < t.b; i += blockDim.x) {
    const long long e = e0 + i;
    float g = 0.f;
    for (int w = 0; w < a.W; ++w)
      if ((wmask >> w) & 1u) g += ld_cg_f(a.vgrads_peer[w] + e);
    float p = a.vparams_local[e];
    step1(e, g, p);
    for (int r = 0; r < a.nranks; ++r) a.vparams_peer[r][e] = p;
  }
}

__device__ __forceinline__ void ps_vec_tile(const PsArgs2& a, const OptC& c, const Unit2& u, const Tile2& t,
                                            unsigned int wmask, bool all_workers, float inv_w) {
  ps_vec_walk(
      a, u, t, wmask, all_workers,
      [&](long long e, const float4& g, float4& p) {
        float4 m = *reinterpret_cast<float4*>(a.vmom + e);
        float4 q = make_float4(0.f, 0.f, 0.f, 0.f), qm = q;
        if (c.opt != OPT_SGD) {
          q = *reinterpret_cast<float4*>(a.vsq + e);
          if (c.opt == OPT_AMSGRAD) qm = *reinterpret_cast<float4*>(a.vsqmax + e);
        }
        opt_update(g.x * inv_w, p.x, m.x, q.x, qm.x, c);
        opt_update(g.y * inv_w, p.y, m.y, q.y, qm.y, c);
        opt_update(g.z * inv_w, p.z, m.z, q.z, qm.z, c);
        opt_update(g.w * inv_w, p.w, m.w, q.w, qm.w, c);
        *reinterpret_cast<float4*>(a.vmom + e) = m;
        if (c.opt != OPT_SGD) {
          *reinterpret_cast<float4*>(a.vsq + e) = q;
          if (c.opt == OPT_AMSGRAD) *reinterpret_cast<float4*>(a.vsqmax + e) = qm;
        }
      },
      [&](long long e, float g, float& p) {
        float m = a.vmom[e], q = 0.f, qm = 0.f;
        if (c.opt != OPT_SGD) { q = a.vsq[e]; if (c.opt == OPT_AMSGRAD) qm = a.vsqmax[e]; }
        opt_update(g * inv_w, p, m, q, qm, c);
        a.vmom[e] = m;
        if (c.opt != OPT_SGD) { a.vsq[e] = q; if (c.opt == OPT_AMSGRAD) a.vsqmax[e] = qm; }
      });
}

// Lion: the same walk, the Lion step on vparams / vmom (vectors take no weight decay)
__device__ __forceinline__ void ps_vec_tile(const PsArgsLion& a, const OptC& c, const Unit2& u, const Tile2& t,
                                            unsigned int wmask, bool all_workers, float inv_w) {
  ps_vec_walk(
      a, u, t, wmask, all_workers,
      [&](long long e, const float4& g, float4& p) {
        float4 m = *reinterpret_cast<float4*>(a.vmom + e);
        lion_update(g.x * inv_w, p.x, m.x, c);
        lion_update(g.y * inv_w, p.y, m.y, c);
        lion_update(g.z * inv_w, p.z, m.z, c);
        lion_update(g.w * inv_w, p.w, m.w, c);
        *reinterpret_cast<float4*>(a.vmom + e) = m;
      },
      [&](long long e, float g, float& p) {
        float m = a.vmom[e];
        lion_update(g * inv_w, p, m, c);
        a.vmom[e] = m;
      });
}

// layer-wise: vectors take momentum-SGD (LARS) or Adam (LAMB) without weight decay and trust ratio
__device__ __forceinline__ void ps_vec_tile(const PsArgsLw& a, const OptC& c, const Unit2& u, const Tile2& t,
                                            unsigned int wmask, bool all_workers, float inv_w) {
  OptC cv = c;
  cv.opt = c.opt == OPT_LARS ? OPT_SGD : OPT_ADAM;
  cv.wd = 0.f;
  ps_vec_tile(static_cast<const PsArgs2&>(a), cv, u, t, wmask, all_workers, inv_w);
}

// gather: the vector tile's mean gradient into vgrad, its squares into the thread's partial (the sums as ps_vec_tile)
__device__ __forceinline__ void ps_vec_tile(const PsArgsGather& a, const OptC&, const Unit2& u, const Tile2& t,
                                            unsigned int wmask, bool all_workers, float inv_w) {
  const int tid = threadIdx.x;
  const long long e0 = u.w_off + t.a;
  const int nvec = t.b >> 2;
  float acc = lw_acc[tid].x;
  for (int v = tid; v < nvec; v += blockDim.x) {
    const long long e = e0 + 4LL * v;
    float4 g;
    if (a.vgrads_mc != nullptr && all_workers) {
      g = multimem_ld_reduce_f4(reinterpret_cast<const float4*>(a.vgrads_mc + e));
    } else {
      g = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int w = 0; w < a.W; ++w) {
        if (!((wmask >> w) & 1u)) continue;
        const float4 x = ld_cg_f4(reinterpret_cast<const float4*>(a.vgrads_peer[w] + e));
        g.x += x.x; g.y += x.y; g.z += x.z; g.w += x.w;
      }
    }
    g = make_float4(g.x * inv_w, g.y * inv_w, g.z * inv_w, g.w * inv_w);
    acc = fmaf(g.x, g.x, acc); acc = fmaf(g.y, g.y, acc); acc = fmaf(g.z, g.z, acc); acc = fmaf(g.w, g.w, acc);
    *reinterpret_cast<float4*>(a.vgrad + e) = g;
  }
  for (int i = (nvec << 2) + tid; i < t.b; i += blockDim.x) {
    const long long e = e0 + i;
    float g = 0.f;
    for (int w = 0; w < a.W; ++w)
      if ((wmask >> w) & 1u) g += ld_cg_f(a.vgrads_peer[w] + e);
    g *= inv_w;
    acc = fmaf(g, g, acc);
    a.vgrad[e] = g;
  }
  lw_acc[tid].x = acc;
}

// end of vector tile ti: only the gather instantiation keeps a partial of it (every thread of the CTA)
template <class A>
__device__ __forceinline__ void clip_vec_done(const A& a, int ti) {
  if constexpr (ps_gather<A>) lw_tile_done(a, ti);
}

// ---- bf16 weight tile that travels dense: the counted workers' staged copies summed in worker order, optimizer,
// bf16 broadcast.  v2_ps_kernel keeps its own inline copy (calling this there changes its instruction schedule).
template <class A>
__device__ __forceinline__ void ps_dense16_tile(const A& a, const OptC& c, const Unit2& u, const Tile2& t,
                                                unsigned int wmask, float inv_w) {
  const int tid = threadIdx.x;
  const long long e0 = u.w_off + t.a;
  const long long s0 = (long long)u.rs + t.a;
  const int nvec = (((e0 | s0) & 7) == 0) ? (t.b >> 3) : 0;
  for (int v = tid; v < nvec; v += blockDim.x) {
    float g[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = 0.f;
    for (int w = 0; w < a.W; ++w) {
      if (!((wmask >> w) & 1u)) continue;
      const uint4 y = ld_cg_u4(a.stage_peer[w] + s0 + 8LL * v);
      const uint32_t ws[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) { g[2 * i] += bf16_lo(ws[i]); g[2 * i + 1] += bf16_hi(ws[i]); }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] *= inv_w;
    update8(a, c, e0 + 8LL * v, g);
  }
  for (int i = (nvec << 3) + tid; i < t.b; i += blockDim.x) {
    float g = 0.f;
    for (int w = 0; w < a.W; ++w)
      if ((wmask >> w) & 1u) g += ld_cg_bf16(a.stage_peer[w] + s0 + i);
    update1(a, c, e0 + i, g * inv_w);
  }
}

// ---- completion (thread 0 of every CTA): group counter; the last CTA of the final group publishes the
// parameters of `step` (param_flag[owner] = step + 1 on every rank) ---------------------------------------------
__device__ __forceinline__ void ps_complete(const PsArgs2& a, Ctrl2* ctrl, int step, bool bad, long long t_enter,
                                            long long t_ready) {
  if (bad) atomicOr(&ctrl->error, ERR2_SLOT_STEP);
  __threadfence_system();
  const unsigned int old = atomicAdd(a.group_counter, 1u);
  if (old == gridDim.x - 1) {
    *a.group_counter = 0;
    __threadfence_system();
    if (a.final_group)
      for (int r = 0; r < a.nranks; ++r) st_release_sys(a.sig_peer[r] + SIG_PARAM + a.owner, step + 1);
    if (a.tstats != nullptr) {
      const long long now = globaltimer_ns();
      a.tstats[0] += t_ready - t_enter;
      a.tstats[1] += now - t_ready;
      a.tstats[2] += 1;
      if (a.final_group) a.tstats[7] += now - a.tstats[6];   // step start -> this owner's parameters published
    }
  }
}

// ---- host: the arguments of a PS launch (the atomo_v2_launch_ps* parameters, in order) and its grid ------------
inline PsArgs2 ps_args(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                       int final_group, int owner, float* master, float* mom, float* sq, float* sqmax, float* vmom,
                       float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer, float* vparams_local,
                       float* vparams_mc, float* const* vparams_peer, const float* vgrads_mc,
                       const float* const* vgrads_peer, const void* const* stage_peer, const float* arenas,
                       long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                       unsigned int* group_counter, long long timeout, long long* tstats, float inv_w) {
  PsArgs2 a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.ntiles = ntiles; a.W = W; a.nranks = nranks;
  a.group = group; a.final_group = final_group; a.owner = owner; a.master = master; a.mom = mom; a.sq = sq;
  a.sqmax = sqmax; a.vmom = vmom; a.vsq = vsq; a.vsqmax = vsqmax; a.wshadow_mc = (__nv_bfloat16*)wshadow_mc;
  a.wshadow_peer = (__nv_bfloat16* const*)wshadow_peer; a.vparams_local = vparams_local; a.vparams_mc = vparams_mc;
  a.vparams_peer = vparams_peer; a.vgrads_mc = vgrads_mc; a.vgrads_peer = vgrads_peer;
  a.stage_peer = (const __nv_bfloat16* const*)stage_peer; a.arenas = arenas; a.arena_floats = arena_floats;
  a.sig = sig; a.sig_peer = sig_peer; a.ctrl = (Ctrl2*)ctrl; a.group_counter = group_counter; a.timeout = timeout;
  a.tstats = tstats; a.inv_w = inv_w;
  return a;
}

// at least one CTA, at most one per tile
inline int ps_grid(int grid, int ntiles) {
  if (grid < 1) grid = 1;
  if (ntiles > 0 && grid > ntiles) grid = ntiles;
  return grid;
}

}  // namespace v2
}  // namespace atomo
