// Layer-wise optimizers of the overlapped / sharded engine (sm_90a): LARS and LAMB, phase 2.
//
// Phase 1 is the layer-wise instantiation of the code's PS kernel (v2_ps_common.cuh, PsArgsLw): it leaves the
// direction x of every weight element it owns in `dir` (LARS: d = g + wd w, LAMB: u) and (sum w^2, sum x^2) per PS
// tile in `part`, and finishes the vector tiles.  This launch, one per group and owner on the PS stream right after
// phase 1:
//   1. sums this owner's tile partials per tensor of the group, in fp64 and tile order;
//   2. with several owners, stores them into every rank's exchange slots of (group, owner), zeros for the tensors it
//      holds no tile of, raises its flag SIG_NORMS + group * MAX_WORKERS + owner = step on every rank, waits for every
//      owner's flag and sums the slots in owner order: every owner gets the same norms bit for bit;
//   3. takes each tensor's trust ratio in fp32: LARS eta ||w|| / (||g|| + wd ||w||), LAMB ||w|| / ||u||, 1 where a norm
//      or the denominator is 0;
//   4. steps its tiles: LARS m = mu m + ratio d (m = ratio d on the first step), w -= lr m; LAMB w -= lr ratio u;
//   5. broadcasts the bf16 weights as update8 does (multimem.st, or the peer loop) and completes through ps_complete
//      with its own group counter (the last group publishes the parameters of the step).
// Every sum runs in a fixed order, so a run is bitwise repeatable and graph replay equals eager.
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int LW_MAX_LAYERS = LW_THREADS;   // weight tensors per group: one thread each for the norms

struct LwArgs : PsArgs2 {
  const int* tile_layer;     // per PS tile of the launch: group-local tensor index, -1 for a vector tile
  int nlayers;
  const float2* part;        // per PS tile of the launch: (sum w^2, sum x^2) of phase 1
  const float* dir;
  double* xch;               // this rank's exchange slots of the group: [2 (step parity)][n_owners][nlayers][2]
  double* const* xch_peer;   // [nranks] the same slots on every rank
  int n_owners;
  float* ratio_out;          // [nlayers] the group's trust ratios (diagnostics; written by CTA 0)
};

__device__ __forceinline__ float lw_step(const OptC& c, float ratio, float x, float p, float& m) {
  if (c.opt == OPT_LARS) {
    m = c.first ? ratio * x : fmaf(c.mu, m, ratio * x);
    return fmaf(-c.lr, m, p);
  }
  return fmaf(-c.lr * ratio, x, p);
}

__global__ void __launch_bounds__(LW_THREADS) v2_layerwise_kernel(const LwArgs a) {
  __shared__ double s_norm[LW_MAX_LAYERS][2];
  __shared__ float s_ratio[LW_MAX_LAYERS];
  __shared__ int s_ok;
  const int tid = threadIdx.x;
  Ctrl2* ctrl = a.ctrl;
  const int step = ctrl->step;
  const long long t_enter = tid == 0 ? globaltimer_ns() : 0;
  const OptC c = ps_opt_consts(ctrl, step);

  // ---- 1. this owner's norms per tensor: fp32 tile partials summed in fp64, in tile order
  if (tid < a.nlayers) {
    double sw = 0.0, sx = 0.0;
    for (int ti = 0; ti < a.ntiles; ++ti) {
      if (a.tile_layer[ti] != tid) continue;
      const float2 p = __ldcg(a.part + ti);
      sw += (double)p.x;
      sx += (double)p.y;
    }
    s_norm[tid][0] = sw;
    s_norm[tid][1] = sx;
  }
  if (tid == 0) s_ok = 1;

  // ---- 2. exchange with the other owners
  if (a.n_owners > 1) {
    const long long par = (long long)(step & 1) * a.n_owners * a.nlayers * 2;
    if (blockIdx.x == 0 && tid < a.nlayers)
      for (int r = 0; r < a.nranks; ++r) {
        double* slot = a.xch_peer[r] + par + ((long long)a.owner * a.nlayers + tid) * 2;
        slot[0] = s_norm[tid][0];
        slot[1] = s_norm[tid][1];
      }
    __syncthreads();
    if (tid == 0) {
      if (blockIdx.x == 0) {
        __threadfence_system();   // the slots before the flag
        for (int r = 0; r < a.nranks; ++r)
          st_release_sys(a.sig_peer[r] + SIG_NORMS + a.group * MAX_WORKERS + a.owner, step);
      }
      bool ok = true;
      for (int o = 0; o < a.n_owners; ++o)
        ok = spin_wait_ge(a.sig + SIG_NORMS + a.group * MAX_WORKERS + o, step, a.timeout) && ok;
      if (!ok) atomicOr(&ctrl->error, ERR2_WAIT_NORMS);
      s_ok = ok ? 1 : 0;
    }
    __syncthreads();
    if (tid < a.nlayers) {
      double sw = 0.0, sx = 0.0;
      for (int o = 0; o < a.n_owners; ++o) {
        const double* slot = a.xch + par + ((long long)o * a.nlayers + tid) * 2;
        sw += __ldcg(slot);
        sx += __ldcg(slot + 1);
      }
      s_norm[tid][0] = sw;
      s_norm[tid][1] = sx;
    }
  }

  // ---- 3. trust ratios, in fp32
  if (tid < a.nlayers) {
    const float wn = sqrtf((float)s_norm[tid][0]), xn = sqrtf((float)s_norm[tid][1]);
    float ratio = 1.f;
    if (c.opt == OPT_LARS) {
      const float den = fmaf(c.wd, wn, xn);
      if (wn > 0.f && den > 0.f) ratio = __fdiv_rn(ctrl->trust_coefficient * wn, den);
    } else if (wn > 0.f && xn > 0.f) {
      ratio = __fdiv_rn(wn, xn);
    }
    s_ratio[tid] = ratio;
    if (blockIdx.x == 0 && a.ratio_out != nullptr) a.ratio_out[tid] = ratio;
  }
  __syncthreads();

  // ---- 4. + 5. step the tiles of this CTA, broadcast bf16
  const auto [t_begin, t_end] = ps_tile_range(a);
  for (int ti = t_begin; s_ok && ti < t_end; ++ti) {
    const int layer = a.tile_layer[ti];
    if (layer < 0) continue;
    const Tile2 t = a.tiles[ti];
    const LwSegs sg = lw_tile_segs(a.units[t.unit], t);
    const float ratio = s_ratio[layer];
    if (((sg.seglen | sg.segbase | sg.segstride) & 7) == 0) {
      const int spv = sg.seglen >> 3;
      for (int v = tid; v < sg.nseg * spv; v += blockDim.x) {
        const int s = v / spv, i8 = v - s * spv;
        const long long e = sg.segbase + s * sg.segstride + 8LL * i8;
        float p[8], x[8], m[8];
        *reinterpret_cast<float4*>(p) = *reinterpret_cast<const float4*>(a.master + e);
        *reinterpret_cast<float4*>(p + 4) = *reinterpret_cast<const float4*>(a.master + e + 4);
        *reinterpret_cast<float4*>(x) = *reinterpret_cast<const float4*>(a.dir + e);
        *reinterpret_cast<float4*>(x + 4) = *reinterpret_cast<const float4*>(a.dir + e + 4);
        if (c.opt == OPT_LARS) {
          *reinterpret_cast<float4*>(m) = *reinterpret_cast<const float4*>(a.mom + e);
          *reinterpret_cast<float4*>(m + 4) = *reinterpret_cast<const float4*>(a.mom + e + 4);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) p[i] = lw_step(c, ratio, x[i], p[i], m[i]);
        *reinterpret_cast<float4*>(a.master + e) = *reinterpret_cast<const float4*>(p);
        *reinterpret_cast<float4*>(a.master + e + 4) = *reinterpret_cast<const float4*>(p + 4);
        if (c.opt == OPT_LARS) {
          *reinterpret_cast<float4*>(a.mom + e) = *reinterpret_cast<const float4*>(m);
          *reinterpret_cast<float4*>(a.mom + e + 4) = *reinterpret_cast<const float4*>(m + 4);
        }
        const uint4 packed = pack_bf16x8(p);
        if (a.wshadow_mc != nullptr) {
          mc_store16(a.wshadow_mc + e, packed);
        } else {
          for (int r = 0; r < a.nranks; ++r) *reinterpret_cast<uint4*>(a.wshadow_peer[r] + e) = packed;
        }
      }
    } else {
      for (int v = tid; v < sg.nseg * sg.seglen; v += blockDim.x) {
        const int s = v / sg.seglen, i = v - s * sg.seglen;
        const long long e = sg.segbase + s * sg.segstride + i;
        float m = c.opt == OPT_LARS ? a.mom[e] : 0.f;
        const float p = lw_step(c, ratio, a.dir[e], a.master[e], m);
        a.master[e] = p;
        if (c.opt == OPT_LARS) a.mom[e] = m;
        const __nv_bfloat16 b = __float2bfloat16_rn(p);
        for (int r = 0; r < a.nranks; ++r) a.wshadow_peer[r][e] = b;
      }
    }
  }

  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, false, t_enter, t_enter);
}

// the PS kernels' layer-wise instantiations (v2_ps.cu, v2_qsgd.cu, v2_entrywise.cu, v2_sign.cu, v2_fp8.cu,
// v2_hadamard.cu, v2_powersgd.cu)
extern "C" {
void atomo_v2_launch_ps_spectral_lw(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_qsgd_lw(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_entry_lw(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_sign_lw(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_fp8_lw(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_hadamard_lw(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_powersgd_lw(const void* args, int grid, cudaStream_t stream);

int atomo_v2_layerwise_max_layers() { return LW_MAX_LAYERS; }

// phase 1: `ps` selects the PS kernel of the code (0 spectral / dense, 1 QSGD / TernGrad, 2 entry-wise / top-k,
// 3 sign, 4 fp8, 5 hadamard, 6 PowerSGD); `part` is already offset to the launch's first tile
void atomo_v2_launch_ps_layerwise(int ps, const void* units, const void* tiles, int tile0, int ntiles, int W,
                                  int nranks, int group, int owner, float* master, float* mom, float* sq, float* vmom,
                                  float* vsq, float* vparams_local, float* vparams_mc, float* const* vparams_peer,
                                  const float* vgrads_mc, const float* const* vgrads_peer,
                                  const void* const* stage_peer, const float* arenas, long long arena_floats, int* sig,
                                  int* const* sig_peer, void* ctrl, unsigned int* group_counter, long long timeout,
                                  long long* tstats, float inv_w, float* dir, void* part, int grid,
                                  cudaStream_t stream) {
  PsArgsLw a;
  static_cast<PsArgs2&>(a) =
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, 0, owner, master, mom, sq, nullptr, vmom, vsq, nullptr,
              nullptr, nullptr, vparams_local, vparams_mc, vparams_peer, vgrads_mc, vgrads_peer, stage_peer, arenas,
              arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w);
  a.dir = dir;
  a.part = static_cast<float2*>(part);
  switch (ps) {
    case 0: atomo_v2_launch_ps_spectral_lw(&a, grid, stream); break;
    case 1: atomo_v2_launch_ps_qsgd_lw(&a, grid, stream); break;
    case 2: atomo_v2_launch_ps_entry_lw(&a, grid, stream); break;
    case 3: atomo_v2_launch_ps_sign_lw(&a, grid, stream); break;
    case 4: atomo_v2_launch_ps_fp8_lw(&a, grid, stream); break;
    case 5: atomo_v2_launch_ps_hadamard_lw(&a, grid, stream); break;
    default: atomo_v2_launch_ps_powersgd_lw(&a, grid, stream); break;
  }
}

// phase 2; tile_layer / part are offset to the launch's first tile, xch to the group's slots (xch_peer: [nranks]
// pointers to them), ratio_out to the group's first tensor
void atomo_v2_launch_layerwise(const void* units, const void* tiles, int tile0, int ntiles, const int* tile_layer,
                               int nlayers, const void* part, const float* dir, int nranks, int group, int final_group,
                               int owner, int n_owners, float* master, float* mom, void* wshadow_mc,
                               void* const* wshadow_peer, double* xch, double* const* xch_peer, int* sig,
                               int* const* sig_peer, void* ctrl, unsigned int* group_counter, long long timeout,
                               long long* tstats, float* ratio_out, int grid, cudaStream_t stream) {
  LwArgs a;
  static_cast<PsArgs2&>(a) =
      ps_args(units, tiles, tile0, ntiles, 0, nranks, group, final_group, owner, master, mom, nullptr, nullptr, nullptr,
              nullptr, nullptr, wshadow_mc, wshadow_peer, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
              nullptr, 0, sig, sig_peer, ctrl, group_counter, timeout, tstats, 0.f);
  a.tile_layer = tile_layer;
  a.nlayers = nlayers;
  a.part = static_cast<const float2*>(part);
  a.dir = dir;
  a.xch = xch;
  a.xch_peer = xch_peer;
  a.n_owners = n_owners;
  a.ratio_out = ratio_out;
  v2_layerwise_kernel<<<ps_grid(grid, ntiles), LW_THREADS, 0, stream>>>(a);
}
}  // extern "C"

}  // namespace v2
}  // namespace atomo
