// Parameter-server side of the overlapped / sharded engine (sm_90a): one launch per backward group and owner.
//
// Reference (SURVEY.md 2.5 K2/K7/K8/K9): rank 0 alone waits for P x (W-1) pickles, decodes each with two
// np.dot calls (codings/svd.py:173), accumulates in float64, steps the optimizer (optim/sgd.py:57-90,
// optim/adam.py:37-94) and re-broadcasts every tensor with one MPI.Bcast each (master:173-279).
//
// Here every GPU owns 1/n_owners of the tiles of each group ("sharded PS"; n_owners = 1 reproduces the
// centralized PS).  As soon as the W step-stamped push flags of a group are visible (ld.acquire.sys on the
// owner's own HBM, written by the workers' project kernels over NVLink) the owner
//   * low-rank tile : gathers the W workers' factors of the tile from its arena, G = (1/W) Ucat (S V)cat
//                     with 4x4 register tiles (K = sum_w count_w ~ 3 W is tiny: bytes, not FLOPs, bound this),
//   * dense tile    : fp32 vectors through multimem.ld_reduce (in-switch NVLS sum of the workers' gradient
//                     buffers), bf16 weights that travel dense from the workers' staging regions,
//   * fused epilogue: weight decay + momentum-SGD / Adam / AMSGrad on the fp32 master copy that exists only
//                     here, rounding to bf16 and ONE multimem.st per 16 bytes that the switch replicates into
//                     every rank's working copy of the weights (layout = the layout cuDNN consumes),
//   * the last CTA of the last group publishes param_flag[owner] = step + 1 on every rank.
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int PS2_THREADS = 256;
constexpr int PS2_KC = 32;
constexpr int PS2_TILE_ELEMS = 4608;
constexpr int PS2_MAX_ROWS = 256;
constexpr int PS2_UP = PS2_MAX_ROWS + 4;   // row pitch of the transposed U chunk
constexpr int PS2_SMEM = (PS2_TILE_ELEMS + PS2_KC * V2_MAX_COLS + PS2_KC * PS2_UP) * 4;

extern __shared__ __align__(16) float ps2_smem[];

template <class A>
__device__ __forceinline__ void ps_spectral(const A& a) {
  float* OUT = ps2_smem;                         // tile of the averaged gradient, physical element order
  float* SV = OUT + PS2_TILE_ELEMS;              // [PS2_KC][64]
  float* UT = SV + PS2_KC * V2_MAX_COLS;         // [PS2_KC][PS2_UP]  (transposed U chunk)
  __shared__ int cnt[MAX_WORKERS], koff[MAX_WORKERS + 1];
  __shared__ int grp_w[MAX_WORKERS * V2_RCAP_MAX / 4], grp_a0[MAX_WORKERS * V2_RCAP_MAX / 4];
  __shared__ int s_ngrp, s_ok, s_bad;

  const int tid = threadIdx.x;
  Ctrl2* ctrl = a.ctrl;
  const int step = ctrl->step;

  // ---- 1. wait for the pushes of this group ------------------------------------------------------------
  // Default: all W workers.  With Ctrl2::num_aggregate = N < W (the reference's --num-aggregate, parsed at
  // distributed_nn.py:67 and never used there) the owner proceeds as soon as N pushes of THIS step have landed:
  // CTA 0 decides the set once and publishes it (mask, then a step stamp) so that every CTA of the launch
  // averages the same workers; late pushes carry an older step in their flag and are simply never counted.
  __shared__ unsigned int s_mask;
  long long t_enter = 0, t_ready = 0;
  if (tid == 0) {
    t_enter = globaltimer_ns();
    bool ok = true;
    const int* flags = a.sig + SIG_PUSH + a.group * MAX_WORKERS;
    const int need = (ctrl->num_aggregate > 0 && ctrl->num_aggregate < a.W) ? ctrl->num_aggregate : a.W;
    unsigned int mask = a.W >= 32 ? 0xffffffffu : ((1u << a.W) - 1u);
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
    if (!ok) atomicOr(&ctrl->error, ERR2_WAIT_PUSH);
    s_ok = ok ? 1 : 0;
    s_bad = 0;
    s_mask = mask;
    t_ready = globaltimer_ns();
  }
  __syncthreads();
  const bool ok = s_ok != 0;
  const unsigned int wmask = s_mask;
  const bool all_workers = wmask == (a.W >= 32 ? 0xffffffffu : ((1u << a.W) - 1u));

  OptC c;
  c.lr = ctrl->lr; c.mu = ctrl->momentum; c.damp = ctrl->dampening; c.wd = ctrl->weight_decay;
  c.nesterov = ctrl->nesterov; c.first = (step == ctrl->first_step); c.opt = ctrl->opt;
  c.b1 = ctrl->beta1; c.b2 = ctrl->beta2; c.eps = ctrl->eps;
  {
    const float t = (float)(step - ctrl->first_step + 1);
    c.bc1 = 1.f - powf(c.b1, t);
    c.sbc2 = sqrtf(1.f - powf(c.b2, t));
  }
  const float inv_w = all_workers ? a.inv_w : 1.f / (float)max(__popc(wmask), 1);

  const int per_cta = (a.ntiles + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta;
  const int t_end = min(a.ntiles, t_begin + per_cta);
  lw_begin(a);
  for (int ti = t_begin; ok && ti < t_end; ++ti) {
    const Tile2 t = a.tiles[ti];
    const Unit2 u = a.units[t.unit];

    if (u.kind == KIND_VEC) {
      // ---------------------------------------------------------------- fp32 vectors (BN, biases)
      ps_vec_tile(a, c, u, t, wmask, all_workers, inv_w);
      clip_vec_done(a, ti);
      continue;
    }

    if (u.kind == KIND_DENSE16) {
      // ---------------------------------------------------------------- bf16 weights that travel dense
      const long long e0 = u.w_off + t.a;
      const long long s0 = (long long)u.rs + t.a;
      const bool vec = ((e0 | s0) & 7) == 0;
      const int nvec = vec ? (t.b >> 3) : 0;
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
      lw_tile_done(a, ti);
      continue;
    }

    // ------------------------------------------------------------------ low-rank tile (K2)
    const int n = u.cols, rcap = u.rcap;
    const int row0 = t.a, nrows = t.b;
    const int nrq = (nrows + 3) >> 2, ncg = (n + 3) >> 2, ncp = ncg << 2;
    __syncthreads();   // previous tile is done with shared memory
    if (tid < a.W) {
      const int* hdr = reinterpret_cast<const int*>(a.arenas + (long long)tid * a.arena_floats + u.slot_off);
      int cc = 0;
      if ((wmask >> tid) & 1u) {
        cc = ld_cg_i(hdr);
        if (ld_cg_i(hdr + 1) != step) { cc = 0; s_bad = 1; }   // stale slot: a push of another step
      }
      cnt[tid] = min(max(cc, 0), rcap);
    }
    __syncthreads();
    if (tid == 0) {
      int k = 0, g = 0;
      for (int w = 0; w < a.W; ++w) {
        koff[w] = k; k += cnt[w];
        for (int a0 = 0; a0 < cnt[w]; a0 += 4) { grp_w[g] = w; grp_a0[g] = a0; ++g; }
      }
      koff[a.W] = k;
      s_ngrp = g;
    }
    __syncthreads();
    const int Ktot = koff[a.W], NG = s_ngrp;
    // physical mapping of (local row r, column c) inside the tile
    const int half = u.I >> 1;
    for (int k0 = 0; k0 < max(Ktot, 1); k0 += PS2_KC) {
      const int kc = min(PS2_KC, Ktot - k0);
      if (k0 > 0) __syncthreads();
      for (int e = tid; e < kc * ncp; e += blockDim.x) {
        const int k = e / ncp, cc = e - k * ncp;
        const int kk = k0 + k;
        int w = 0;
        while (kk >= koff[w + 1]) ++w;
        const int at = kk - koff[w];
        const float* slot = a.arenas + (long long)w * a.arena_floats + u.slot_off;
        float v = 0.f;
        if (cc < n) v = ld_cg_f(slot + 4 + at) * ld_cg_f(slot + 4 + rcap + (long long)at * n + cc);
        SV[k * V2_MAX_COLS + cc] = v;
      }
      for (int e = tid; e < kc * (4 * nrq - nrows); e += blockDim.x) {   // zero the row padding
        const int k = e / (4 * nrq - nrows), r = nrows + e - k * (4 * nrq - nrows);
        UT[k * PS2_UP + r] = 0.f;
      }
      for (int e = tid; e < nrows * NG; e += blockDim.x) {
        const int g = e / nrows, r = e - g * nrows;
        const int w = grp_w[g], a0 = grp_a0[g];
        const int kbase = koff[w] + a0 - k0;
        if (kbase >= kc || kbase + 4 <= 0) continue;
        const float* slotw = a.arenas + (long long)w * a.arena_floats + u.slot_off;
        const float* U = slotw + slot2_u_off(rcap, n);
        float uv[4];
        if (u.ubits == 8) {   // QSVD: 4 x int8 and the row scale
          const int q = ld_cg_i(reinterpret_cast<const int*>(U) + (((long long)(row0 + r) * rcap + a0) >> 2));
          const float sc = ld_cg_f(slotw + slot2_scale_off(u.rows, rcap, n) + row0 + r) * (1.f / 127.f);
#pragma unroll
          for (int j = 0; j < 4; ++j) uv[j] = (float)(signed char)((q >> (8 * j)) & 0xff) * sc;
        } else {
          const float4 u4 = ld_cg_f4(reinterpret_cast<const float4*>(U + (long long)(row0 + r) * rcap + a0));
          uv[0] = u4.x; uv[1] = u4.y; uv[2] = u4.z; uv[3] = u4.w;
        }
        const int lim = cnt[w] - a0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = kbase + j;
          if (j < lim && k >= 0 && k < kc) UT[k * PS2_UP + r] = uv[j];
        }
      }
      __syncthreads();
      for (int it = tid; it < nrq * ncg; it += blockDim.x) {
        const int cg = it / nrq, rq = it - cg * nrq;
        float acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
        for (int k = 0; k < kc; ++k) {
          const float4 uu = *reinterpret_cast<const float4*>(&UT[k * PS2_UP + 4 * rq]);
          const float4 sv = *reinterpret_cast<const float4*>(&SV[k * V2_MAX_COLS + 4 * cg]);
          const float ur[4] = {uu.x, uu.y, uu.z, uu.w}, sc[4] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ur[i], sc[j], acc[i][j]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = 4 * rq + i;
          if (r >= nrows) continue;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int cc = 4 * cg + j;
            if (cc >= n) continue;
            int o;
            if (u.kind == KIND_SLAB) {
              const int s = r / half, ri = r - s * half;
              const int b = cc >= u.K ? 1 : 0, k = cc - b * u.K;
              o = (s * u.K + k) * u.I + 2 * ri + b;
            } else if (u.cs == 1) {
              o = r * n + cc;
            } else {
              o = cc * nrows + r;
            }
            const float val = acc[i][j] * inv_w;
            OUT[o] = (k0 == 0) ? val : OUT[o] + val;
          }
        }
      }
    }
    __syncthreads();

    // ---- fused optimizer epilogue + bf16 parameter broadcast ------------------------------------
    int nseg, seglen;
    long long segbase, segstride;
    if (u.kind == KIND_SLAB) {
      nseg = 1; seglen = (nrows / half) * u.K * u.I; segbase = u.w_off + (long long)(row0 / half) * u.K * u.I; segstride = 0;
    } else if (u.cs == 1) {
      nseg = nrows; seglen = n; segbase = u.w_off + (long long)row0 * u.rs; segstride = u.rs;
    } else {
      nseg = n; seglen = nrows; segbase = u.w_off + row0; segstride = u.cs;
    }
    const bool vec = ((seglen | segbase | segstride) & 7) == 0;
    if (vec) {
      const int spv = seglen >> 3;
      for (int v = tid; v < nseg * spv; v += blockDim.x) {
        const int s = v / spv, i8 = v - s * spv;
        const float4 g0 = *reinterpret_cast<const float4*>(&OUT[s * seglen + 8 * i8]);
        const float4 g1 = *reinterpret_cast<const float4*>(&OUT[s * seglen + 8 * i8 + 4]);
        const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        update8(a, c, segbase + s * segstride + 8LL * i8, g);
      }
    } else {
      for (int v = tid; v < nseg * seglen; v += blockDim.x) {
        const int s = v / seglen, i = v - s * seglen;
        update1(a, c, segbase + s * segstride + i, OUT[v]);
      }
    }
    lw_tile_done(a, ti);
  }

  // ---- completion ------------------------------------------------------------------------------------
  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, s_bad != 0, t_enter, t_ready);
}

__global__ void __launch_bounds__(PS2_THREADS) v2_ps_kernel(const PsArgs2 a) { ps_spectral(a); }
__global__ void __launch_bounds__(PS2_THREADS, 1) v2_ps_lw_kernel(const PsArgsLw a) { ps_spectral(a); }
__global__ void __launch_bounds__(PS2_THREADS, 1) v2_ps_gather_kernel(const PsArgsGather a) { ps_spectral(a); }
__global__ void __launch_bounds__(PS2_THREADS, 1) v2_ps_lion_kernel(const PsArgsLion a) { ps_spectral(a); }

// worker side: block the stream until every owner has delivered its shard of the parameters of `step`
__global__ void v2_wait_params_kernel(const int* sig, int n_owners, Ctrl2* ctrl, long long timeout, long long* tstats) {
  const long long t0 = globaltimer_ns();
  if ((int)threadIdx.x < n_owners) {
    if (!spin_wait_ge(sig + SIG_PARAM + threadIdx.x, ctrl->step, timeout)) atomicOr(&ctrl->error, ERR2_WAIT_PARAM);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // a straggler that was left out of an aggregation (num_aggregate < W) finds the owners already further along:
    // it skips ahead to the step whose parameters are in place instead of pushing gradients nobody waits for
    int m = 0x7fffffff;
    for (int o = 0; o < n_owners; ++o) m = min(m, ld_acquire_sys(sig + SIG_PARAM + o));
    if (m != 0x7fffffff && m > ctrl->step) ctrl->step = m;
  }
  if (threadIdx.x == 0 && tstats != nullptr) {
    const long long now = globaltimer_ns();
    tstats[3] += now - t0; tstats[4] += 1;
    tstats[6] = now;                                             // step start stamp
  }
}

__global__ void v2_advance_step_kernel(Ctrl2* ctrl) {
  if (threadIdx.x == 0) ctrl->step += 1;
}

// initial sync / checkpoint load: copy `n16` 16-byte words of the local region to every rank
__global__ void v2_bcast_bytes_kernel(const uint4* __restrict__ src, uint4* const* peer, uint4* mc, int nranks, int self,
                                      long long n16) {
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n16; v += (long long)gridDim.x * blockDim.x) {
    const uint4 x = src[v];
    if (mc != nullptr) {
      mc_store16(mc + v, x);
    } else {
      for (int r = 0; r < nranks; ++r)
        if (r != self) peer[r][v] = x;
    }
  }
}

extern "C" {

int atomo_v2_ps_smem() { return PS2_SMEM; }
int atomo_v2_ps_tile_elems() { return PS2_TILE_ELEMS; }

void atomo_v2_launch_ps(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                        int final_group, int owner, float* master, float* mom, float* sq, float* sqmax, float* vmom,
                        float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer, float* vparams_local,
                        float* vparams_mc, float* const* vparams_peer, const float* vgrads_mc,
                        const float* const* vgrads_peer, const void* const* stage_peer, const float* arenas,
                        long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                        unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                        cudaStream_t stream) {
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(v2_ps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PS2_SMEM);
    attr = true;
  }
  v2_ps_kernel<<<ps_grid(grid, ntiles), PS2_THREADS, PS2_SMEM, stream>>>(
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, final_group, owner, master, mom, sq, sqmax, vmom, vsq,
              vsqmax, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, vgrads_mc, vgrads_peer,
              stage_peer, arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w));
}

void atomo_v2_launch_ps_spectral_lw(const void* args, int grid, cudaStream_t stream) {
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(v2_ps_lw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PS2_SMEM);
    attr = true;
  }
  const PsArgsLw& a = *static_cast<const PsArgsLw*>(args);
  v2_ps_lw_kernel<<<ps_grid(grid, a.ntiles), PS2_THREADS, PS2_SMEM, stream>>>(a);
}

void atomo_v2_launch_ps_spectral_gather(const void* args, int grid, cudaStream_t stream) {
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(v2_ps_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PS2_SMEM);
    attr = true;
  }
  const PsArgsGather& a = *static_cast<const PsArgsGather*>(args);
  v2_ps_gather_kernel<<<ps_grid(grid, a.ntiles), PS2_THREADS, PS2_SMEM, stream>>>(a);
}

void atomo_v2_launch_ps_spectral_lion(const void* args, int grid, cudaStream_t stream) {
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(v2_ps_lion_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PS2_SMEM);
    attr = true;
  }
  const PsArgsLion& a = *static_cast<const PsArgsLion*>(args);
  v2_ps_lion_kernel<<<ps_grid(grid, a.ntiles), PS2_THREADS, PS2_SMEM, stream>>>(a);
}

void atomo_v2_launch_wait_params(const int* sig, int n_owners, void* ctrl, long long timeout, long long* tstats,
                                 cudaStream_t stream) {
  v2_wait_params_kernel<<<1, 32, 0, stream>>>(sig, n_owners, (Ctrl2*)ctrl, timeout, tstats);
}
void atomo_v2_launch_advance_step(void* ctrl, cudaStream_t stream) {
  v2_advance_step_kernel<<<1, 32, 0, stream>>>((Ctrl2*)ctrl);
}
void atomo_v2_launch_bcast_bytes(const void* src, void* const* peer, void* mc, int nranks, int self, long long nbytes,
                                 cudaStream_t stream) {
  const long long n16 = nbytes / 16;
  int grid = (int)((n16 + 255) / 256);
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  if (grid < 1) grid = 1;
  v2_bcast_bytes_kernel<<<grid, 256, 0, stream>>>((const uint4*)src, (uint4* const*)peer, (uint4*)mc, nranks, self, n16);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
