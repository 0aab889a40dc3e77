// K2/K7/K8/K9 — parameter-server side, one persistent kernel (sm_90a).
//
// Reference pipeline (SURVEY.md 2.5 K2/K7/K8/K9, call stack 3.2): MPI waitany over
// P x (W-1) pickles -> np.dot(np.dot(u, diag(s)), vT) per (layer, worker)
// (codings/svd.py:173) -> float64 += (master:292-296) -> /(W-1) (master:238) ->
// optim.SGD.step (optim/sgd.py:57-90) -> next step: one float64 MPI.Bcast per
// tensor (master:270-279) + step handshake (master:246-252).
//
// Here: ONE kernel on the PS GPU.  Each persistent CTA
//   1. acquires the W workers' step-stamped push flags (ld.acquire.sys spin on
//      its own HBM; the flags were written by peers over NVLink)          [C6]
//   2. walks a tile table.  Low-rank tile: gathers the W workers' factors from
//      the arenas (written by K1's peer stores), forms the K = sum_w count_w
//      concatenated rank-1 terms, reconstructs the averaged gradient tile
//      G = (1/W) * Ucat * (S V)cat in registers/shared memory.  Dense tile:
//      G = (1/W) sum_w grad_w read from the workers' gradient buffers through
//      NVLink (multimem.ld_reduce in-switch sum when NVLS is bound, else peer
//      loads)                                                              [K7]
//   3. fused epilogue: weight decay + momentum + Nesterov + p -= lr*d      [optim/sgd.py]
//   4. broadcasts the updated parameter tile to every rank: one
//      multimem.st per 16 bytes (NVLS replicates it) or per-peer stores    [K8, C3/C4]
//   5. the last CTA publishes param_flag = step+1 on every rank            [K9, C1/C2]
// No NCCL, no host round trip, no per-tensor launches.
#include "common.cuh"

namespace atomo {

constexpr int PS_THREADS = 256;
constexpr int PS_KC = 32;           // K chunk (concatenated atoms) staged per iteration
constexpr int PS_TILE_ELEMS = 4096; // output elements per low-rank tile (rows*cols <= this)
constexpr int PS_MAX_ROWS = 256;
constexpr int PS_MAX_W = 16;
constexpr int PS_DENSE_ELEMS = 4096;

struct PsArgs {
  const LayerDesc* layers;
  const TileDesc* tiles;
  int ntiles;
  int W;               // number of gradient sources (arenas / gradient buffers)
  int nflags;          // push flags to wait for before touching any source
  int nranks;          // ranks receiving parameters
  float* params;       // local flat parameters
  float* momentum;     // local momentum buffer (PS only)
  float* const* params_peer;      // [nranks] peer pointers to every rank's flat parameters (incl. self)
  float* params_mc;               // NVLS multicast alias of the parameter buffer (or nullptr)
  const float* const* grads_peer; // [W] peer pointers to the workers' flat gradient buffers
  const float* grads_mc;          // NVLS multicast alias of the gradient buffers (or nullptr)
  const float* arenas;            // local: worker w's factors live at arenas + w*arena_floats
  long long arena_floats;
  int* push_flags;                // local [W]
  int* const* param_flag_peer;    // [nranks] pointer to each rank's param flag
  Ctrl* ctrl;
  long long timeout_ticks;
  float inv_w;                    // 1 / (number of gradients averaged)
  long long* tstats;              // optional device stats: [0] sum ns waiting for pushes, [1] sum ns working, [2] steps
};

__device__ __forceinline__ void sgd_update(float g, float& p, float& m, const float lr, const float mu,
                                           const float damp, const float wd, const int nesterov,
                                           const bool first) {
  g = fmaf(wd, p, g);
  float d = g;
  if (mu != 0.f) {
    m = first ? g : fmaf(mu, m, (1.f - damp) * g);
    d = nesterov ? fmaf(mu, m, g) : m;
  }
  p = fmaf(-lr, d, p);
}

__device__ __forceinline__ void bcast_store4(const PsArgs& a, long long e, const float4 v) {
  if (a.params_mc != nullptr) {
    multimem_st_f4(reinterpret_cast<float4*>(a.params_mc + e), v);
  } else {
    for (int r = 0; r < a.nranks; ++r) st_na_f4(reinterpret_cast<float4*>(a.params_peer[r] + e), v);
  }
}
__device__ __forceinline__ void bcast_store1(const PsArgs& a, long long e, const float v) {
  // scalar tail / unaligned layouts: unicast peer stores (multimem.st needs vectors to be worthwhile)
  for (int r = 0; r < a.nranks; ++r) a.params_peer[r][e] = v;
}

extern __shared__ __align__(16) float ps_smem[];

__global__ void __launch_bounds__(PS_THREADS)
ps_update_kernel(PsArgs a) {
  // dynamic shared memory carve-up
  float* OUT = ps_smem;                                  // PS_TILE_ELEMS
  float* SV = OUT + PS_TILE_ELEMS;                       // PS_KC x 64
  float* UT = SV + PS_KC * TS_MAX_COLS;                  // PS_MAX_ROWS x (PS_KC+1)
  __shared__ int cnt[PS_MAX_W], koff[PS_MAX_W + 1];
  __shared__ int grp_w[PS_MAX_W * RCAP_MAX / 4], grp_a0[PS_MAX_W * RCAP_MAX / 4];
  __shared__ int s_ngrp;
  __shared__ int s_ok;

  const int tid = threadIdx.x;
  Ctrl* ctrl = a.ctrl;
  const int step = ctrl->step;

  // ---- 1. wait for every worker's push of this step ------------------------------------
  long long t_enter = 0, t_ready = 0;
  if (tid == 0) {
    t_enter = globaltimer_ns();
    bool ok = true;
    for (int w = 0; w < a.nflags; ++w) ok = spin_wait_ge(a.push_flags + w, step, a.timeout_ticks) && ok;
    if (!ok) atomicExch(&ctrl->error, ERR_WAIT_PUSH_TIMEOUT);
    s_ok = ok ? 1 : 0;
    t_ready = globaltimer_ns();
  }
  __syncthreads();
  const bool ok = s_ok != 0;

  const float lr = ctrl->lr, mu = ctrl->momentum, damp = ctrl->dampening, wd = ctrl->weight_decay;
  const int nesterov = ctrl->nesterov;
  const bool first = (step == ctrl->first_step);
  const float inv_w = a.inv_w;

  // contiguous tile ranges per CTA: consecutive tiles mostly belong to the same layer, so the
  // per-layer factor table (counts, S*V) is staged once and reused
  const int per_cta = (a.ntiles + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta;
  const int t_end = min(a.ntiles, t_begin + per_cta);
  int cached_layer = -1, cached_col0 = -1;
  for (int ti = t_begin; ok && ti < t_end; ++ti) {
    const TileDesc t = a.tiles[ti];
    const LayerDesc L = a.layers[t.layer];

    if (L.route == ROUTE_DENSE) {
      // ------------------------------------------------------------ dense tile (K7)
      const long long e0 = L.off + (long long)t.row0 * 4;
      const int nelem = t.nrows;
      const int nvec = nelem >> 2;
      for (int v = tid; v < nvec; v += blockDim.x) {
        const long long e = e0 + 4LL * v;
        float4 g;
        if (a.grads_mc != nullptr) {
          g = multimem_ld_reduce_f4(reinterpret_cast<const float4*>(a.grads_mc + e));
        } else {
          g = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int w = 0; w < a.W; ++w) {
            const float4 x = ld_cg_f4(reinterpret_cast<const float4*>(a.grads_peer[w] + e));
            g.x += x.x; g.y += x.y; g.z += x.z; g.w += x.w;
          }
        }
        float4 p = *reinterpret_cast<float4*>(a.params + e);
        float4 m = *reinterpret_cast<float4*>(a.momentum + e);
        sgd_update(g.x * inv_w, p.x, m.x, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.y * inv_w, p.y, m.y, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.z * inv_w, p.z, m.z, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.w * inv_w, p.w, m.w, lr, mu, damp, wd, nesterov, first);
        *reinterpret_cast<float4*>(a.momentum + e) = m;
        bcast_store4(a, e, p);
      }
      for (int i = (nvec << 2) + tid; i < nelem; i += blockDim.x) {  // tail (< 4 elements)
        const long long e = e0 + i;
        float g = 0.f;
        for (int w = 0; w < a.W; ++w) g += ld_cg_f(a.grads_peer[w] + e);
        float p = a.params[e], m = a.momentum[e];
        sgd_update(g * inv_w, p, m, lr, mu, damp, wd, nesterov, first);
        a.momentum[e] = m;
        bcast_store1(a, e, p);
      }
      continue;
    }

    // ---------------------------------------------------------------- low-rank tile (K2)
    const int n = L.cols;
    const int col0 = t.col0;
    const int nc = min(TS_MAX_COLS, n - col0);  // columns handled by this tile
    const int nc4 = (nc + 3) >> 2;
    const int ncp = nc4 << 2;
    const int rows = t.nrows;
    const int rcap = L.rcap;
    const bool same = (t.layer == cached_layer && col0 == cached_col0);

    __syncthreads();  // previous tile fully consumed shared memory
    if (!same) {
      if (tid < a.W) {
        const int* hdr = reinterpret_cast<const int*>(a.arenas + (long long)tid * a.arena_floats + L.slot_off);
        int c = ld_cg_i(hdr);
        cnt[tid] = min(max(c, 0), rcap);
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
    }
    const int K = koff[a.W];
    const int NG = s_ngrp;
    const bool single = K <= PS_KC;

    // accumulators: items (row, 4-column group); up to 4 items per thread
    const int items = rows * nc4;
    float4 acc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);

    for (int k0 = 0; k0 < K; k0 += PS_KC) {
      const int kc = min(PS_KC, K - k0);
      if (k0 > 0) __syncthreads();
      // SV[k][c] = s_w[a] * V_w[a][col0 + c]   (kept across tiles of the same layer when K fits one chunk)
      if (!(same && single)) {
        for (int e = tid; e < kc * ncp; e += blockDim.x) {
          const int k = e / ncp, c = e - k * ncp;
          const int kk = k0 + k;
          int w = 0;
          while (kk >= koff[w + 1]) ++w;
          const int at = kk - koff[w];
          const float* slot = a.arenas + (long long)w * a.arena_floats + L.slot_off;
          float v = 0.f;
          if (c < nc) v = ld_cg_f(slot + slot_s_off() + at) * ld_cg_f(slot + slot_v_off(rcap) + (long long)at * n + col0 + c);
          SV[k * TS_MAX_COLS + c] = v;
        }
      }
      // UT[r][k] = U_w[row0 + r][a]: one 16-byte load per (row, worker, 4-atom group)
      for (int e = tid; e < rows * NG; e += blockDim.x) {
        const int r = e / NG, g = e - r * NG;
        const int w = grp_w[g], a0 = grp_a0[g];
        const int kbase = koff[w] + a0 - k0;   // position of atom a0 inside this chunk
        if (kbase >= kc || kbase + 4 <= 0) continue;
        const float* U = a.arenas + (long long)w * a.arena_floats + L.slot_off + slot_u_off(rcap, n);
        const float4 u4 = ld_cg_f4(reinterpret_cast<const float4*>(U + (long long)(t.row0 + r) * rcap + a0));
        const float uv[4] = {u4.x, u4.y, u4.z, u4.w};
        const int lim = cnt[w] - a0;  // atoms of this group that exist
        float* dst = &UT[r * (PS_KC + 1)];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = kbase + j;
          if (j < lim && k >= 0 && k < kc) dst[k] = uv[j];
        }
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int it = tid + i * PS_THREADS;
        if (it < items) {
          const int r = it / nc4, cg = it - r * nc4;
          const float* ur = &UT[r * (PS_KC + 1)];
          for (int k = 0; k < kc; ++k) {
            const float u = ur[k];
            const float4 sv = *reinterpret_cast<const float4*>(&SV[k * TS_MAX_COLS + 4 * cg]);
            acc[i].x = fmaf(u, sv.x, acc[i].x); acc[i].y = fmaf(u, sv.y, acc[i].y);
            acc[i].z = fmaf(u, sv.z, acc[i].z); acc[i].w = fmaf(u, sv.w, acc[i].w);
          }
        }
      }
    }
    cached_layer = single ? t.layer : -1;
    cached_col0 = col0;
    __syncthreads();
    // stage the averaged gradient tile: OUT[r*nc + c]
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int it = tid + i * PS_THREADS;
      if (it < items) {
        const int r = it / nc4, cg = it - r * nc4;
        const float v4[4] = {acc[i].x, acc[i].y, acc[i].z, acc[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = 4 * cg + j;
          if (c < nc) OUT[r * nc + c] = v4[j] * inv_w;
        }
      }
    }
    __syncthreads();

    // fused optimizer epilogue + parameter broadcast
    if (L.vec_ok == 1 && nc == n) {
      // the tile is one contiguous, 16-byte aligned run of rows*n floats
      const long long e0 = L.off + (long long)t.row0 * n;
      const int nvec = (rows * n) >> 2;
      for (int v = tid; v < nvec; v += blockDim.x) {
        const long long e = e0 + 4LL * v;
        const float4 g = *reinterpret_cast<const float4*>(&OUT[4 * v]);
        float4 p = *reinterpret_cast<float4*>(a.params + e);
        float4 m = *reinterpret_cast<float4*>(a.momentum + e);
        sgd_update(g.x, p.x, m.x, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.y, p.y, m.y, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.z, p.z, m.z, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.w, p.w, m.w, lr, mu, damp, wd, nesterov, first);
        *reinterpret_cast<float4*>(a.momentum + e) = m;
        bcast_store4(a, e, p);
      }
      for (int i = (nvec << 2) + tid; i < rows * n; i += blockDim.x) {
        const long long e = e0 + i;
        float p = a.params[e], m = a.momentum[e];
        sgd_update(OUT[i], p, m, lr, mu, damp, wd, nesterov, first);
        a.momentum[e] = m;
        bcast_store1(a, e, p);
      }
    } else if (L.vec_ok == 2 && (nc & 3) == 0) {
      // column-tiled wide layer: every row segment [col0, col0+nc) is contiguous and 16-byte aligned
      const int q4 = nc >> 2;
      for (int i = tid; i < rows * q4; i += blockDim.x) {
        const int r = i / q4, c4 = i - r * q4;
        const long long e = L.off + (long long)(t.row0 + r) * L.row_stride + col0 + 4 * c4;
        const float4 g = *reinterpret_cast<const float4*>(&OUT[r * nc + 4 * c4]);
        float4 p = *reinterpret_cast<float4*>(a.params + e);
        float4 m = *reinterpret_cast<float4*>(a.momentum + e);
        sgd_update(g.x, p.x, m.x, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.y, p.y, m.y, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.z, p.z, m.z, lr, mu, damp, wd, nesterov, first);
        sgd_update(g.w, p.w, m.w, lr, mu, damp, wd, nesterov, first);
        *reinterpret_cast<float4*>(a.momentum + e) = m;
        bcast_store4(a, e, p);
      }
    } else if (L.vec_ok == 3 && (rows & 3) == 0 && (t.row0 & 3) == 0) {
      // transposed orientation: memory is contiguous along the tall rows
      const int r4n = rows >> 2;
      for (int i = tid; i < nc * r4n; i += blockDim.x) {
        const int c = i / r4n, r4 = i - c * r4n;
        const long long e = L.off + (long long)(t.row0 + 4 * r4) * L.row_stride + (long long)(col0 + c) * L.col_stride;
        const float* o = &OUT[(4 * r4) * nc + c];
        float4 p = *reinterpret_cast<float4*>(a.params + e);
        float4 m = *reinterpret_cast<float4*>(a.momentum + e);
        sgd_update(o[0], p.x, m.x, lr, mu, damp, wd, nesterov, first);
        sgd_update(o[nc], p.y, m.y, lr, mu, damp, wd, nesterov, first);
        sgd_update(o[2 * nc], p.z, m.z, lr, mu, damp, wd, nesterov, first);
        sgd_update(o[3 * nc], p.w, m.w, lr, mu, damp, wd, nesterov, first);
        *reinterpret_cast<float4*>(a.momentum + e) = m;
        bcast_store4(a, e, p);
      }
    } else {
      for (int i = tid; i < rows * nc; i += blockDim.x) {
        int r, c;
        if (L.col_stride == 1) { r = i / nc; c = i - r * nc; }
        else { c = i / rows; r = i - c * rows; }  // keep consecutive threads on consecutive addresses
        const long long e = L.off + (long long)(t.row0 + r) * L.row_stride + (long long)(col0 + c) * L.col_stride;
        float p = a.params[e], m = a.momentum[e];
        sgd_update(OUT[r * nc + c], p, m, lr, mu, damp, wd, nesterov, first);
        a.momentum[e] = m;
        bcast_store1(a, e, p);
      }
    }
  }

  // ---- 5. completion: the last CTA tells every rank "parameters of step+1 are in place" ----
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    const unsigned int old = atomicAdd(&ctrl->done_ps, 1u);
    if (old == gridDim.x - 1) {
      ctrl->done_ps = 0;
      __threadfence_system();
      for (int r = 0; r < a.nranks; ++r) st_release_sys(a.param_flag_peer[r], step + 1);
      if (a.tstats != nullptr) {  // the last CTA to finish closes the books for this step
        a.tstats[0] += t_ready - t_enter;
        a.tstats[1] += globaltimer_ns() - t_ready;
        a.tstats[2] += 1;
      }
    }
  }
}

// worker side of K9: block the stream until the PS has delivered the parameters of `step`
__global__ void wait_params_kernel(const int* param_flag, Ctrl* ctrl, long long timeout_ticks, long long* tstats) {
  if (threadIdx.x == 0) {
    const long long t0 = globaltimer_ns();
    if (!spin_wait_ge(param_flag, ctrl->step, timeout_ticks)) atomicExch(&ctrl->error, ERR_WAIT_PARAM_TIMEOUT);
    if (tstats != nullptr) { tstats[3] += globaltimer_ns() - t0; tstats[4] += 1; }
  }
}

__global__ void advance_step_kernel(Ctrl* ctrl) {
  if (threadIdx.x == 0) ctrl->step += 1;
}

// K8 alone: broadcast the local flat parameter buffer to every rank (initial sync, checkpoint load)
__global__ void param_bcast_kernel(const float* __restrict__ src, float* const* params_peer, float* params_mc,
                                   int nranks, int self_rank, long long n4) {
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n4;
       v += (long long)gridDim.x * blockDim.x) {
    const float4 x = reinterpret_cast<const float4*>(src)[v];
    if (params_mc != nullptr) {
      multimem_st_f4(reinterpret_cast<float4*>(params_mc) + v, x);
    } else {
      for (int r = 0; r < nranks; ++r)
        if (r != self_rank) st_na_f4(reinterpret_cast<float4*>(params_peer[r]) + v, x);
    }
  }
}

__global__ void set_flags_kernel(int* const* flag_peer, int nranks, int value) {
  if (threadIdx.x == 0) {
    __threadfence_system();
    for (int r = 0; r < nranks; ++r) st_release_sys(flag_peer[r], value);
  }
}

// ----------------------------------------------------------------------------
extern "C" {

int atomo_ps_smem_bytes() { return (PS_TILE_ELEMS + PS_KC * TS_MAX_COLS + PS_MAX_ROWS * (PS_KC + 1)) * 4; }
int atomo_ps_tile_elems() { return PS_TILE_ELEMS; }
int atomo_ps_max_rows() { return PS_MAX_ROWS; }
int atomo_ps_dense_elems() { return PS_DENSE_ELEMS; }
int atomo_ps_max_workers() { return PS_MAX_W; }

void atomo_launch_ps_update(const void* layers, const void* tiles, int ntiles, int W, int nflags, int nranks,
                            float* params,
                            float* momentum, float* const* params_peer, float* params_mc,
                            const float* const* grads_peer, const float* grads_mc, const float* arenas,
                            long long arena_floats, int* push_flags, int* const* param_flag_peer, void* ctrl,
                            long long timeout_ticks, float inv_w, int grid, long long* tstats, cudaStream_t stream) {
  static bool attr_set = false;
  const int smem = atomo_ps_smem_bytes();
  if (!attr_set) {
    cudaFuncSetAttribute(ps_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr_set = true;
  }
  PsArgs a;
  a.layers = (const LayerDesc*)layers; a.tiles = (const TileDesc*)tiles; a.ntiles = ntiles; a.W = W;
  a.nflags = nflags;
  a.nranks = nranks; a.params = params; a.momentum = momentum; a.params_peer = params_peer;
  a.params_mc = params_mc; a.grads_peer = grads_peer; a.grads_mc = grads_mc; a.arenas = arenas;
  a.arena_floats = arena_floats; a.push_flags = push_flags; a.param_flag_peer = param_flag_peer;
  a.ctrl = (Ctrl*)ctrl; a.timeout_ticks = timeout_ticks; a.inv_w = inv_w; a.tstats = tstats;
  if (grid < 1) grid = 1;
  ps_update_kernel<<<grid, PS_THREADS, smem, stream>>>(a);
}

void atomo_launch_wait_params(const int* param_flag, void* ctrl, long long timeout_ticks, long long* tstats,
                              cudaStream_t stream) {
  wait_params_kernel<<<1, 32, 0, stream>>>(param_flag, (Ctrl*)ctrl, timeout_ticks, tstats);
}

void atomo_launch_advance_step(void* ctrl, cudaStream_t stream) {
  advance_step_kernel<<<1, 32, 0, stream>>>((Ctrl*)ctrl);
}

void atomo_launch_param_bcast(const float* src, float* const* params_peer, float* params_mc, int nranks,
                              int self_rank, long long numel, cudaStream_t stream) {
  const long long n4 = numel / 4;
  int grid = (int)((n4 + 255) / 256);
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  if (grid < 1) grid = 1;
  param_bcast_kernel<<<grid, 256, 0, stream>>>(src, params_peer, params_mc, nranks, self_rank, n4);
}

void atomo_launch_set_flags(int* const* flag_peer, int nranks, int value, cudaStream_t stream) {
  set_flags_kernel<<<1, 32, 0, stream>>>(flag_peer, nranks, value);
}

}  // extern "C"
}  // namespace atomo
