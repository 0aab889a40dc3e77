// Gradient-norm clipping on the overlapped / sharded engine (sm_90a): phase 2, one launch per owner and step.
//
// Phase 1 is the gather instantiation of the code's PS kernel (v2_ps_common.cuh, PsArgsGather), one launch per group:
// it leaves the mean gradient g of every element it owns in `grad` / `vgrad` and sum g^2 per PS tile in `gpart`.
// This launch, on the PS stream right after the final group's phase 1:
//   1. sums this owner's tile partials of the whole step in fp64: thread t takes tiles t, t + 256, ... of the owner's
//      tile list in order, then a fixed tree over the CTA (every CTA computes the same sum);
//   2. with several owners, stores it into every rank's slot (step parity, owner), raises SIG_CLIP + owner = step on
//      every rank, waits for every owner's flag and sums the slots in owner order: every owner gets the same norm
//      bit for bit;
//   3. total = ||g||, coef = min(1, max_norm / (total + 1e-6)) as torch.nn.utils.clip_grad_norm_ (a NaN stays NaN);
//      a non-finite total sets ERR2_NONFINITE;
//   4. steps every tile of the owner on coef * g:
//      - SGD / Adam / AMSGrad: through update8 / update1 (the plain PS epilogue, bf16 broadcast included) and the
//        vector optimizer with its fp32 broadcast; completes through ps_complete with final_group = 1, so this launch
//        publishes the parameters of the step;
//      - LARS / LAMB: through the layer-wise update8 / update1 (direction into `dir`, which is `grad` itself, and
//        (w^2, x^2) per PS tile into `lwpart`), vectors finished as layer-wise phase 1 does; v2_layerwise.cu then runs
//        per group as without clipping, and its last launch publishes.
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int CLIP_THREADS = LW_THREADS;

struct ClipArgs : PsArgsLw {    // PsArgsLw::dir / part: LARS / LAMB's direction and tile partials (else unused)
  const int* owner_tiles;       // this owner's PS tiles of every group, in group order (ntiles of them)
  const float2* gpart;          // per PS tile: (sum g^2, 0) of phase 1
  const float* grad;            // g, indexed like master
  const float* vgrad;           // g of the vector tiles, indexed like vparams
  double* xch;                  // this rank's exchange slots: [2 (step parity)][n_owners]
  double* const* xch_peer;      // [nranks] the same slots on every rank
  int n_owners;
  float* norm_out;              // [2]: total, coef (written by CTA 0)
};

// one vector tile on coef * g: the optimizer and fp32 broadcast of ps_vec_tile
__device__ __forceinline__ void clip_vec_tile(const ClipArgs& a, const OptC& c, const Unit2& u, const Tile2& t,
                                              float coef) {
  const int tid = threadIdx.x;
  const long long e0 = u.w_off + t.a;
  const int nvec = t.b >> 2;
  for (int v = tid; v < nvec; v += blockDim.x) {
    const long long e = e0 + 4LL * v;
    const float4 g = __ldcg(reinterpret_cast<const float4*>(a.vgrad + e));
    float4 p = *reinterpret_cast<float4*>(a.vparams_local + e);
    float4 m = *reinterpret_cast<float4*>(a.vmom + e);
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f), qm = q;
    if (c.opt != OPT_SGD) {
      q = *reinterpret_cast<float4*>(a.vsq + e);
      if (c.opt == OPT_AMSGRAD) qm = *reinterpret_cast<float4*>(a.vsqmax + e);
    }
    opt_update(g.x * coef, p.x, m.x, q.x, qm.x, c);
    opt_update(g.y * coef, p.y, m.y, q.y, qm.y, c);
    opt_update(g.z * coef, p.z, m.z, q.z, qm.z, c);
    opt_update(g.w * coef, p.w, m.w, q.w, qm.w, c);
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
    float p = a.vparams_local[e], m = a.vmom[e], q = 0.f, qm = 0.f;
    if (c.opt != OPT_SGD) { q = a.vsq[e]; if (c.opt == OPT_AMSGRAD) qm = a.vsqmax[e]; }
    opt_update(__ldcg(a.vgrad + e) * coef, p, m, q, qm, c);
    a.vmom[e] = m;
    if (c.opt != OPT_SGD) { a.vsq[e] = q; if (c.opt == OPT_AMSGRAD) a.vsqmax[e] = qm; }
    for (int r = 0; r < a.nranks; ++r) a.vparams_peer[r][e] = p;
  }
}

// one weight tile on coef * g through A's epilogue (PsArgs2: optimizer + bf16 broadcast; PsArgsLw: direction +
// partials), in the element order of lw_tile_segs
template <class A>
__device__ __forceinline__ void clip_weight_tile(const ClipArgs& a, const A& ea, const OptC& c, const Unit2& u,
                                                 const Tile2& t, float coef) {
  const int tid = threadIdx.x;
  const LwSegs sg = lw_tile_segs(u, t);
  if (((sg.seglen | sg.segbase | sg.segstride) & 7) == 0) {
    const int spv = sg.seglen >> 3;
    for (int v = tid; v < sg.nseg * spv; v += blockDim.x) {
      const int s = v / spv, i8 = v - s * spv;
      const long long e = sg.segbase + s * sg.segstride + 8LL * i8;
      float g[8];
      *reinterpret_cast<float4*>(g) = __ldcg(reinterpret_cast<const float4*>(a.grad + e));
      *reinterpret_cast<float4*>(g + 4) = __ldcg(reinterpret_cast<const float4*>(a.grad + e + 4));
#pragma unroll
      for (int i = 0; i < 8; ++i) g[i] *= coef;
      update8(ea, c, e, g);
    }
  } else {
    for (int v = tid; v < sg.nseg * sg.seglen; v += blockDim.x) {
      const int s = v / sg.seglen, i = v - s * sg.seglen;
      const long long e = sg.segbase + s * sg.segstride + i;
      update1(ea, c, e, __ldcg(a.grad + e) * coef);
    }
  }
}

template <bool LW>
__device__ __forceinline__ void clip_step(const ClipArgs& a) {
  __shared__ double s_red[CLIP_THREADS];
  __shared__ float s_coef;
  __shared__ int s_ok;
  const int tid = threadIdx.x;
  Ctrl2* ctrl = a.ctrl;
  const int step = ctrl->step;
  const long long t_enter = tid == 0 ? globaltimer_ns() : 0;
  const OptC c = ps_opt_consts(ctrl, step);

  // ---- 1. this owner's sum of g^2: a fixed-order fp64 sum per thread, then a fixed tree
  double s = 0.0;
  for (int i = tid; i < a.ntiles; i += CLIP_THREADS) s += (double)__ldcg(&a.gpart[a.owner_tiles[i]].x);
  s_red[tid] = s;
  __syncthreads();
#pragma unroll
  for (int o = CLIP_THREADS / 2; o > 0; o >>= 1) {
    if (tid < o) s_red[tid] += s_red[tid + o];
    __syncthreads();
  }

  // ---- 2. + 3. exchange with the other owners, the norm and the coefficient (thread 0)
  if (tid == 0) {
    double sum = s_red[0];
    bool ok = true;
    if (a.n_owners > 1) {
      const long long par = (long long)(step & 1) * a.n_owners;
      if (blockIdx.x == 0) {
        for (int r = 0; r < a.nranks; ++r) a.xch_peer[r][par + a.owner] = sum;
        __threadfence_system();   // the slots before the flag
        for (int r = 0; r < a.nranks; ++r) st_release_sys(a.sig_peer[r] + SIG_CLIP + a.owner, step);
      }
      for (int o = 0; o < a.n_owners; ++o) ok = spin_wait_ge(a.sig + SIG_CLIP + o, step, a.timeout) && ok;
      if (!ok) atomicOr(&ctrl->error, ERR2_WAIT_NORMS);
      sum = 0.0;
      for (int o = 0; o < a.n_owners; ++o) sum += __ldcg(a.xch + par + o);
    }
    const float total = (float)sqrt(sum);
    float coef = __fdiv_rn(ctrl->clip_grad_norm, __fadd_rn(total, 1e-6f));
    if (coef > 1.f) coef = 1.f;
    if (blockIdx.x == 0) {
      if (!isfinite(total)) atomicOr(&ctrl->error, ERR2_NONFINITE);
      if (a.norm_out != nullptr) { a.norm_out[0] = total; a.norm_out[1] = coef; }
    }
    s_coef = coef;
    s_ok = ok ? 1 : 0;
  }
  __syncthreads();
  const float coef = s_coef;

  // ---- 4. step this CTA's share of the owner's tiles
  OptC cv = c;      // vectors: LARS -> momentum-SGD, LAMB -> Adam, without weight decay (layer-wise phase 1)
  if constexpr (LW) {
    cv.opt = c.opt == OPT_LARS ? OPT_SGD : OPT_ADAM;
    cv.wd = 0.f;
  }
  const auto [t_begin, t_end] = ps_tile_range(a);
  const PsArgsLw& lwa = a;
  if constexpr (LW) lw_begin(lwa);
  for (int i = t_begin; s_ok && i < t_end; ++i) {
    const int ti = a.owner_tiles[i];
    const Tile2 t = a.tiles[ti];
    const Unit2 u = a.units[t.unit];
    if (u.kind == KIND_VEC) {
      clip_vec_tile(a, cv, u, t, coef);
      continue;
    }
    if constexpr (LW) {
      clip_weight_tile(a, lwa, c, u, t, coef);
      lw_tile_done(lwa, ti);
    } else {
      clip_weight_tile(a, static_cast<const PsArgs2&>(a), c, u, t, coef);
    }
  }

  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, false, t_enter, t_enter);
}

__global__ void __launch_bounds__(CLIP_THREADS) v2_clip_kernel(const ClipArgs a) { clip_step<false>(a); }
__global__ void __launch_bounds__(CLIP_THREADS) v2_clip_lw_kernel(const ClipArgs a) { clip_step<true>(a); }

// the PS kernels' gather instantiations (v2_ps.cu, v2_qsgd.cu, v2_entrywise.cu, v2_sign.cu, v2_fp8.cu,
// v2_hadamard.cu, v2_powersgd.cu)
extern "C" {
void atomo_v2_launch_ps_spectral_gather(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_qsgd_gather(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_entry_gather(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_sign_gather(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_fp8_gather(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_hadamard_gather(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_powersgd_gather(const void* args, int grid, cudaStream_t stream);

// phase 1: `ps` selects the PS kernel of the code (0 spectral / dense, 1 QSGD / TernGrad, 2 entry-wise / top-k,
// 3 sign, 4 fp8, 5 hadamard, 6 PowerSGD); `part` is already offset to the launch's first tile
void atomo_v2_launch_ps_gather(int ps, const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks,
                               int group, int owner, const float* vgrads_mc, const float* const* vgrads_peer,
                               const void* const* stage_peer, const float* arenas, long long arena_floats, int* sig,
                               int* const* sig_peer, void* ctrl, unsigned int* group_counter, long long timeout,
                               long long* tstats, float inv_w, float* grad, float* vgrad, void* part, int grid,
                               cudaStream_t stream) {
  PsArgsGather a;
  static_cast<PsArgs2&>(a) =
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, 0, owner, nullptr, nullptr, nullptr, nullptr, nullptr,
              nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, vgrads_mc, vgrads_peer, stage_peer,
              arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w);
  a.grad = grad;
  a.vgrad = vgrad;
  a.part = static_cast<float2*>(part);
  switch (ps) {
    case 0: atomo_v2_launch_ps_spectral_gather(&a, grid, stream); break;
    case 1: atomo_v2_launch_ps_qsgd_gather(&a, grid, stream); break;
    case 2: atomo_v2_launch_ps_entry_gather(&a, grid, stream); break;
    case 3: atomo_v2_launch_ps_sign_gather(&a, grid, stream); break;
    case 4: atomo_v2_launch_ps_fp8_gather(&a, grid, stream); break;
    case 5: atomo_v2_launch_ps_hadamard_gather(&a, grid, stream); break;
    default: atomo_v2_launch_ps_powersgd_gather(&a, grid, stream); break;
  }
}

// phase 2; `tiles` is the whole PS tile table, owner_tiles this owner's entries of it; with `layerwise` (LARS / LAMB)
// dir must be `grad` and lwpart the layer-wise tile partials (indexed like the PS tile table)
void atomo_v2_launch_clip(int layerwise, const void* units, const void* tiles, const int* owner_tiles, int ntiles,
                          const void* gpart, const float* grad, const float* vgrad, int nranks, int owner, int n_owners,
                          float* master, float* mom, float* sq, float* sqmax, float* vmom, float* vsq, float* vsqmax,
                          void* wshadow_mc, void* const* wshadow_peer, float* vparams_local, float* vparams_mc,
                          float* const* vparams_peer, float* dir, void* lwpart, double* xch, double* const* xch_peer,
                          int* sig, int* const* sig_peer, void* ctrl, unsigned int* counter, long long timeout,
                          long long* tstats, float* norm_out, int grid, cudaStream_t stream) {
  ClipArgs a;
  static_cast<PsArgs2&>(a) =
      ps_args(units, tiles, 0, ntiles, 0, nranks, 0, layerwise ? 0 : 1, owner, master, mom, sq, sqmax, vmom, vsq,
              vsqmax, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, nullptr, nullptr, nullptr,
              nullptr, 0, sig, sig_peer, ctrl, counter, timeout, tstats, 0.f);
  a.dir = dir;
  a.part = static_cast<float2*>(lwpart);
  a.owner_tiles = owner_tiles;
  a.gpart = static_cast<const float2*>(gpart);
  a.grad = grad;
  a.vgrad = vgrad;
  a.xch = xch;
  a.xch_peer = xch_peer;
  a.n_owners = n_owners;
  a.norm_out = norm_out;
  if (layerwise)
    v2_clip_lw_kernel<<<ps_grid(grid, ntiles), CLIP_THREADS, 0, stream>>>(a);
  else
    v2_clip_kernel<<<ps_grid(grid, ntiles), CLIP_THREADS, 0, stream>>>(a);
}
}  // extern "C"

}  // namespace v2
}  // namespace atomo
