// Parameter-server building blocks shared by the PS kernels of the overlapped / sharded engine: the launch
// arguments, the push wait with the --num-aggregate mask, the fp32 vector tiles and the fused optimizer epilogue
// with its bf16 broadcast.  v2_ps.cu (spectral / dense tiles) and v2_qsgd.cu (quantized tiles) both use them.
#pragma once
#include "v2_common.cuh"

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
  const uint4 packed = pack_bf16x8(p);
  if (a.wshadow_mc != nullptr) {
    mc_store16(a.wshadow_mc + e, packed);
  } else {
    for (int r = 0; r < a.nranks; ++r) *reinterpret_cast<uint4*>(a.wshadow_peer[r] + e) = packed;
  }
}

__device__ __forceinline__ void update1(const PsArgs2& a, const OptC& c, long long e, float g) {
  float p = a.master[e], m = a.mom[e], v = 0.f, vm = 0.f;
  if (c.opt != OPT_SGD) { v = a.sq[e]; if (c.opt == OPT_AMSGRAD) vm = a.sqmax[e]; }
  opt_update(g, p, m, v, vm, c);
  a.master[e] = p; a.mom[e] = m;
  if (c.opt != OPT_SGD) { a.sq[e] = v; if (c.opt == OPT_AMSGRAD) a.sqmax[e] = vm; }
  const __nv_bfloat16 b = __float2bfloat16_rn(p);
  for (int r = 0; r < a.nranks; ++r) a.wshadow_peer[r][e] = b;
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
__device__ __forceinline__ void ps_vec_tile(const PsArgs2& a, const OptC& c, const Unit2& u, const Tile2& t,
                                            unsigned int wmask, bool all_workers, float inv_w) {
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
    float p = a.vparams_local[e], m = a.vmom[e], q = 0.f, qm = 0.f;
    if (c.opt != OPT_SGD) { q = a.vsq[e]; if (c.opt == OPT_AMSGRAD) qm = a.vsqmax[e]; }
    opt_update(g * inv_w, p, m, q, qm, c);
    a.vmom[e] = m;
    if (c.opt != OPT_SGD) { a.vsq[e] = q; if (c.opt == OPT_AMSGRAD) a.vsqmax[e] = qm; }
    for (int r = 0; r < a.nranks; ++r) a.vparams_peer[r][e] = p;
  }
}

// ---- bf16 weight tile that travels dense: the counted workers' staged copies summed in worker order, optimizer,
// bf16 broadcast.  v2_ps_kernel keeps its own inline copy (calling this there changes its instruction schedule).
__device__ __forceinline__ void ps_dense16_tile(const PsArgs2& a, const OptC& c, const Unit2& u, const Tile2& t,
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

}  // namespace v2
}  // namespace atomo
