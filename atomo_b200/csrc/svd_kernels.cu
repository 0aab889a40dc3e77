// K1 — spectral-ATOMO encode fused with the worker->PS push (sm_90a).
//
// Reference pipeline (SURVEY.md 2.5 K1): per tensor, host LAPACK SVD
// (codings/svd.py:95) -> Python Bernoulli loop (svd.py:49-67) -> pickle ->
// MPI isend (distributed_worker.py:330-335).  Here ALL tall-skinny layers of the
// model (every 3x3/5x5 conv, small fc) are encoded by three grouped launches that
// walk a tile table, and the sampled factors are stored straight into the
// parameter server's HBM through NVLink peer pointers:
//
//   gram_kernel      : G_tile = A_tile^T A_tile           (pass 1 over the gradient)
//   eig_sample_kernel: G = sum tiles; V,lambda = Jacobi(G); sigma = sqrt(lambda);
//                      p_i = min(1, r sigma_i / sum sigma) (or water-filled);
//                      Philox Bernoulli / systematic sampling;
//                      header, s_a = sigma_a/p_a and V rows -> PS slot (peer store)
//   project_push     : U[:,a] = A v_a / sigma_a            (pass 2, L2-resident)
//                      float4 peer stores of U into the PS slot; the last CTA
//                      publishes the step-stamped flag with st.release.sys.
//
// Because V is a complete orthonormal basis of the skinny dimension,
// sum_i (A v_i) v_i^T == A exactly, so the estimator is unbiased even when the
// fp32 Gram/Jacobi eigenvectors are only approximately the singular vectors.
#include "common.cuh"

namespace atomo {

constexpr int GRAM_THREADS = 256;
constexpr int GRAM_CHUNK = 64;   // rows staged per iteration
constexpr int EIG_THREADS = 256;
constexpr int PROJ_THREADS = 128;
constexpr int MAX_SWEEPS = 12;

// ----------------------------------------------------------------------------
// stage a chunk of tall rows into shared memory: sm[r*stride + c] = A[row0+r][c]
// ----------------------------------------------------------------------------
__device__ __forceinline__ void load_chunk(const float* __restrict__ grad, const LayerDesc& L, int row0, int nrows,
                                           float* sm, int stride) {
  const int n = L.cols;
  const float* base = grad + L.off;
  if (L.col_stride == 1) {
    // rows are contiguous runs of n floats (row_stride == n for matricized tensors)
    const int total = nrows * n;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
      int r = e / n, c = e - r * n;
      sm[r * stride + c] = __ldg(base + (long long)(row0 + r) * L.row_stride + c);
    }
  } else {
    // transposed orientation: consecutive tall rows are adjacent in memory
    const int total = nrows * n;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
      int c = e / nrows, r = e - c * nrows;
      sm[r * stride + c] = __ldg(base + (long long)(row0 + r) * L.row_stride + (long long)c * L.col_stride);
    }
  }
}

// ----------------------------------------------------------------------------
// pass 1: per-tile Gram matrix
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(GRAM_THREADS)
gram_kernel(const float* __restrict__ grad, const LayerDesc* __restrict__ layers, const TileDesc* __restrict__ tiles,
            float* __restrict__ gpart) {
  __shared__ __align__(16) float sm[GRAM_CHUNK * TS_MAX_COLS];
  __shared__ float red[TS_MAX_COLS * TS_MAX_COLS];

  const TileDesc t = tiles[blockIdx.x];
  const LayerDesc L = layers[t.layer];
  const int n = L.cols;
  const int npad = (n + 3) & ~3;
  const int nb = npad >> 2;
  const int NB = nb * nb;
  const int RG = max(1, (int)blockDim.x / NB);
  const int blk = threadIdx.x % NB;
  const int g = threadIdx.x / NB;
  const bool active = g < RG;
  const int bi = blk / nb, bj = blk - bi * nb;

  for (int i = threadIdx.x; i < GRAM_CHUNK * npad; i += blockDim.x) sm[i] = 0.f;
  for (int i = threadIdx.x; i < npad * npad; i += blockDim.x) red[i] = 0.f;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int r0 = 0; r0 < t.nrows; r0 += GRAM_CHUNK) {
    const int cr = min(GRAM_CHUNK, t.nrows - r0);
    __syncthreads();
    load_chunk(grad, L, t.row0 + r0, cr, sm, npad);
    __syncthreads();
    if (active) {
      for (int r = g; r < cr; r += RG) {
        const float4 a = *reinterpret_cast<const float4*>(&sm[r * npad + 4 * bi]);
        const float4 b = *reinterpret_cast<const float4*>(&sm[r * npad + 4 * bj]);
        const float av[4] = {a.x, a.y, a.z, a.w};
        const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
    }
  }
  __syncthreads();
  if (active) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) atomicAdd(&red[(4 * bi + i) * npad + 4 * bj + j], acc[i][j]);
  }
  __syncthreads();
  float* out = gpart + L.gpart_off + (long long)(blockIdx.x - L.tile0) * n * n;
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    int i = e / n, j = e - i * n;
    out[e] = red[i * npad + j];
  }
}

// ----------------------------------------------------------------------------
// eigen-decomposition + sampling, one CTA per tall-skinny layer
// ----------------------------------------------------------------------------
struct EncodeCfg {
  int rank;           // sparsity budget s (0 -> p = sigma/sigma_max, svd.py:52)
  int random_sample;  // 0 -> keep the top-`rank` atoms (svd.py:109-113)
  int waterfill;      // 0 -> reference single clip, 1 -> paper's water-filling
  int systematic;     // 0 -> independent Bernoulli, 1 -> systematic sampling
  int worker_index;   // index of this worker's arena on the PS
  int use_ext_uniforms;
};

constexpr int GS = TS_MAX_COLS + 1;  // padded row stride of G / V in shared memory

__device__ __forceinline__ void rr_pair(int ne, int rnd, int k, int& p, int& q) {
  // round-robin tournament over `ne` (even) players: ne/2 disjoint pairs per round
  const int m = ne - 1;
  int a, b;
  if (k == 0) { a = rnd % m; b = m; }
  else { a = (rnd + k) % m; b = (rnd - k + m) % m; }
  p = min(a, b); q = max(a, b);
}

__global__ void __launch_bounds__(1024)
eig_sample_kernel(const LayerDesc* __restrict__ layers, const int* __restrict__ ts_layers,
                  const float* __restrict__ gpart, float* __restrict__ vsel, int* __restrict__ selcount,
                  float* __restrict__ sigma_out, float* ps_arena_peer, long long arena_floats, const Ctrl* ctrl,
                  const float* __restrict__ ext_uniforms, EncodeCfg cfg) {
  __shared__ float G[TS_MAX_COLS * GS];
  __shared__ float V[TS_MAX_COLS * GS];
  __shared__ float rc[TS_MAX_COLS / 2], rs[TS_MAX_COLS / 2];
  __shared__ int rp[TS_MAX_COLS / 2], rq[TS_MAX_COLS / 2];
  __shared__ float sig[TS_MAX_COLS], prob[TS_MAX_COLS], uni[TS_MAX_COLS];
  __shared__ int order[TS_MAX_COLS];  // order[k] = index of k-th largest sigma
  __shared__ int sel[RCAP_MAX];
  __shared__ float selscale[RCAP_MAX];
  __shared__ int s_maxrel;
  __shared__ float s_gmax;
  __shared__ int s_count, s_done;

  const int layer_id = ts_layers[blockIdx.x];
  const LayerDesc L = layers[layer_id];
  const int n = L.cols;
  const int tid = threadIdx.x;
  const int step = ctrl->step;

  // ---- G = sum of tile partials (padded to an even size with a zero row/col); V = I ----------
  const int ne = n + (n & 1);
  const int npairs = ne >> 1;
  for (int e = tid; e < ne * ne; e += blockDim.x) {
    const int i = e / ne, j = e - i * ne;
    float s = 0.f;
    if (i < n && j < n) {
      const float* gp = gpart + L.gpart_off + i * n + j;
      for (int t = 0; t < L.ntiles; ++t) s += gp[(long long)t * n * n];
    }
    G[i * GS + j] = s;
    V[i * GS + j] = (i == j) ? 1.f : 0.f;
  }
  __syncthreads();
  // symmetrize (partials are accumulated in different orders for (i,j)/(j,i))
  for (int e = tid; e < n * n; e += blockDim.x) {
    int i = e / n, j = e - i * n;
    if (i < j) {
      float v = 0.5f * (G[i * GS + j] + G[j * GS + i]);
      G[i * GS + j] = v;
      G[j * GS + i] = v;
    }
  }
  __syncthreads();

  // ---- cyclic Jacobi, round-robin (parallel) ordering, fused two-sided update ------------------
  // All ne/2 pairs of a round are disjoint, so G' = J^T G J decomposes into independent 2x2
  // blocks: block (k1,k2) = J_k1^T * G[{p1,q1}][{p2,q2}] * J_k2 — one thread per block, one
  // barrier between "compute rotations" and "apply", none between the row and column halves.
  // The padded dummy index only ever meets zeros, so its rotations are the identity.
  if (tid == 0) {
    float g = 0.f;
    for (int i = 0; i < n; ++i) g = fmaxf(g, fabsf(G[i * GS + i]));
    s_gmax = g;
  }
  __syncthreads();
  const float gmax = s_gmax;
  if (n > 1 && gmax > 0.f) {
    for (int sweep = 0; sweep < MAX_SWEEPS; ++sweep) {
      if (tid == 0) s_maxrel = 0;
      __syncthreads();
      for (int rnd = 0; rnd < ne - 1; ++rnd) {
        if (tid < npairs) {
          int p, q;
          rr_pair(ne, rnd, tid, p, q);
          float c = 1.f, s = 0.f;
          const float apq = G[p * GS + q], app = G[p * GS + p], aqq = G[q * GS + q];
          const float scale = sqrtf(fabsf(app * aqq));
          // rotate unless the coupling is below fp32 noise (relative to the pair and to the spectrum)
          if (fabsf(apq) > 1e-7f * scale && fabsf(apq) > 3e-7f * gmax) {
            const float tau = (aqq - app) / (2.f * apq);
            const float t = (tau >= 0.f ? 1.f : -1.f) / (fabsf(tau) + sqrtf(1.f + tau * tau));
            c = rsqrtf(1.f + t * t);
            s = t * c;
            atomicMax(&s_maxrel, __float_as_int(fabsf(apq) / gmax));
          }
          rp[tid] = p; rq[tid] = q; rc[tid] = c; rs[tid] = s;
        }
        __syncthreads();
        const int nblk = npairs * npairs;
        for (int e = tid; e < nblk + npairs * ne; e += blockDim.x) {
          if (e < nblk) {
            const int k1 = e / npairs, k2 = e - k1 * npairs;
            const int p1 = rp[k1], q1 = rq[k1], p2 = rp[k2], q2 = rq[k2];
            const float c1 = rc[k1], s1 = rs[k1], c2 = rc[k2], s2 = rs[k2];
            const float a = G[p1 * GS + p2], b = G[p1 * GS + q2], c_ = G[q1 * GS + p2], d = G[q1 * GS + q2];
            // left: rows (p1,q1) <- J1^T
            const float ra = c1 * a - s1 * c_, rb = c1 * b - s1 * d;
            const float rc_ = s1 * a + c1 * c_, rd = s1 * b + c1 * d;
            // right: cols (p2,q2) <- J2
            G[p1 * GS + p2] = c2 * ra - s2 * rb;
            G[p1 * GS + q2] = s2 * ra + c2 * rb;
            G[q1 * GS + p2] = c2 * rc_ - s2 * rd;
            G[q1 * GS + q2] = s2 * rc_ + c2 * rd;
          } else {
            const int f = e - nblk;
            const int k = f / ne, i = f - k * ne;
            const int p = rp[k], q = rq[k];
            const float c = rc[k], s = rs[k];
            const float vp = V[i * GS + p], vq = V[i * GS + q];
            V[i * GS + p] = c * vp - s * vq;
            V[i * GS + q] = s * vp + c * vq;
          }
        }
        __syncthreads();
      }
      // quadratic convergence: couplings below 1e-3 at the start of a sweep are ~1e-6 after it.  Every thread reads
      // the shared value BEFORE thread 0 may reset it for the next sweep (else a slow warp can leave the loop alone
      // and desynchronise all later barriers).
      const float mr = __int_as_float(s_maxrel);
      __syncthreads();
      if (mr < 1e-3f) break;
    }
  }
  __syncthreads();

  // ---- singular values, descending order --------------------------------------
  if (tid < n) sig[tid] = sqrtf(fmaxf(G[tid * GS + tid], 0.f));
  __syncthreads();
  if (tid < n) {
    const float me = sig[tid];
    int rank_ = 0;
    for (int j = 0; j < n; ++j) {
      const float o = sig[j];
      rank_ += (o > me) || (o == me && j < tid);
    }
    order[rank_] = tid;
  }
  __syncthreads();

  // ---- inclusion probabilities ---------------------------------------------------
  const int rcap = L.rcap;
  if (tid == 0) {
    float total = 0.f;
    for (int i = 0; i < n; ++i) total += sig[i];
    const float smax = sig[order[0]];
    int count = 0;
    if (!(smax >= 1e-6f)) {
      // degenerate spectrum (svd.py:50-51): send atom 0 with probability 1
      sel[0] = order[0]; selscale[0] = 1.f; count = 1;
      for (int i = 0; i < n; ++i) prob[i] = 0.f;
      prob[order[0]] = 1.f;
      s_done = 1;
    } else if (!cfg.random_sample) {
      const int k = min(min(cfg.rank > 0 ? cfg.rank : n, n), rcap);
      for (int a = 0; a < k; ++a) { sel[a] = order[a]; selscale[a] = 1.f; }
      count = k;
      s_done = 1;
    } else {
      if (cfg.rank == 0) {
        for (int i = 0; i < n; ++i) prob[i] = fminf(sig[i] / smax, 1.f);
      } else if (!cfg.waterfill) {
        for (int i = 0; i < n; ++i) prob[i] = fminf((float)cfg.rank * sig[i] / total, 1.f);
      } else {
        // water-filling over the sorted spectrum: pin the largest atoms to 1
        float budget = fminf((float)cfg.rank, (float)n);
        float rest = total;
        int pinned = 0;
        while (pinned < n) {
          const float s0 = sig[order[pinned]];
          if (rest > 0.f && (budget - pinned) * s0 >= rest && (budget - pinned) > 0.f) {
            rest -= s0; ++pinned;
          } else break;
        }
        for (int k = 0; k < n; ++k) {
          const int i = order[k];
          prob[i] = (k < pinned) ? 1.f : (rest > 0.f ? fminf((budget - pinned) * sig[i] / rest, 1.f) : 0.f);
        }
      }
      s_done = 0;
    }
    s_count = count;
  }
  __syncthreads();

  // ---- sampling ----------------------------------------------------------------------
  if (!s_done) {
    for (int attempt = 0; attempt < 16 && !s_done; ++attempt) {
      if (tid < n) {
        float u;
        if (cfg.use_ext_uniforms && attempt == 0) {
          u = ext_uniforms[(long long)blockIdx.x * TS_MAX_COLS + tid];
        } else {
          uint32_t r4[4];
          Philox::gen(ctrl->seed, (uint32_t)tid, (uint32_t)attempt, (uint32_t)layer_id,
                      ((uint32_t)cfg.worker_index << 24) ^ (uint32_t)step, r4);
          u = Philox::to_uniform(r4[0]);
        }
        uni[tid] = u;
      }
      __syncthreads();
      if (tid == 0) {
        int count = 0;
        bool overflow = false;
        if (cfg.systematic) {
          // one uniform, cumulative probabilities in descending-sigma order
          const float u = uni[0];
          float c = 0.f;
          for (int k = 0; k < n; ++k) {
            const int i = order[k];
            const float lo = floorf(c + u);
            c += prob[i];
            const float hi = floorf(c + u);
            if (hi > lo) {
              if (count < rcap) { sel[count] = i; selscale[count] = 1.f / prob[i]; }
              else overflow = true;
              ++count;
            }
          }
        } else {
          for (int k = 0; k < n; ++k) {
            const int i = order[k];
            if (uni[i] < prob[i]) {
              if (count < rcap) { sel[count] = i; selscale[count] = 1.f / prob[i]; }
              else overflow = true;
              ++count;
            }
          }
        }
        if (count > 0 && !overflow) { s_count = count; s_done = 1; }  // else resample (svd.py:65-66)
      }
      __syncthreads();
    }
    if (!s_done) {
      // pathological: deterministic fallback on the most probable atoms
      if (tid == 0) {
        const int k = min(max(cfg.rank, 1), min(n, rcap));
        for (int a = 0; a < k; ++a) { sel[a] = order[a]; selscale[a] = 1.f / fmaxf(prob[order[a]], 1e-6f); }
        s_count = k; s_done = 1;
      }
      __syncthreads();
    }
  }
  const int count = s_count;

  // ---- publish: local projection basis + PS slot header / s / V -----------------------
  // vsel[ts][c*RCAP_MAX + a] = V[c][sel_a] / sigma_a   (so  U = A * vsel)
  float* vs = vsel + (long long)blockIdx.x * TS_MAX_COLS * RCAP_MAX;
  for (int e = tid; e < n * RCAP_MAX; e += blockDim.x) {
    const int c = e / RCAP_MAX, a = e - c * RCAP_MAX;
    float v = 0.f;
    if (a < count) {
      const int i = sel[a];
      // a (numerically) null direction has no left vector: emit a zero column instead of 1/0
      v = (sig[i] > 1e-7f * sig[order[0]]) ? V[c * GS + i] / sig[i] : 0.f;
    }
    vs[e] = v;
  }
  if (tid == 0) selcount[blockIdx.x] = count;
  if (sigma_out != nullptr && tid < n) sigma_out[(long long)blockIdx.x * TS_MAX_COLS + tid] = sig[order[tid]];

  float* slot = ps_arena_peer + (long long)cfg.worker_index * arena_floats + L.slot_off;
  if (tid < rcap) slot[slot_s_off() + tid] = (tid < count) ? sig[sel[tid]] * selscale[tid] : 0.f;
  float* vout = slot + slot_v_off(rcap);
  for (int e = tid; e < rcap * n; e += blockDim.x) {
    const int a = e / n, c = e - a * n;
    vout[e] = (a < count) ? V[c * GS + sel[a]] : 0.f;
  }
  if (tid == 0) {
    int* hdr = reinterpret_cast<int*>(slot);
    hdr[0] = count; hdr[1] = step; hdr[2] = n; hdr[3] = L.rows;
  }
  __threadfence_system();
}

// ----------------------------------------------------------------------------
// pass 2: U = A * vsel, stored straight into the PS slot; last CTA raises the flag
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(PROJ_THREADS)
project_push_kernel(const float* __restrict__ grad, const LayerDesc* __restrict__ layers,
                    const TileDesc* __restrict__ tiles, const float* __restrict__ vsel,
                    const int* __restrict__ selcount, float* ps_arena_peer, long long arena_floats,
                    int* push_flag_peer, Ctrl* ctrl, int worker_index, int signal) {
  __shared__ float sm[PROJ_THREADS * (TS_MAX_COLS + 1)];  // one row per thread, odd stride
  __shared__ __align__(16) float vs[TS_MAX_COLS * RCAP_MAX];

  const TileDesc t = tiles[blockIdx.x];
  const LayerDesc L = layers[t.layer];
  const int n = L.cols;
  const int stride = n | 1;
  const int count = selcount[L.ts_index];
  const int rcap = L.rcap;
  const float* vsrc = vsel + (long long)L.ts_index * TS_MAX_COLS * RCAP_MAX;
  for (int e = threadIdx.x; e < n * RCAP_MAX; e += blockDim.x) vs[e] = vsrc[e];

  float* slot = ps_arena_peer + (long long)worker_index * arena_floats + L.slot_off;
  float* U = slot + slot_u_off(rcap, n);
  const int c4 = (count + 3) >> 2;  // float4 groups actually carrying atoms

  for (int r0 = 0; r0 < t.nrows; r0 += PROJ_THREADS) {
    const int cr = min((int)PROJ_THREADS, t.nrows - r0);
    __syncthreads();
    load_chunk(grad, L, t.row0 + r0, cr, sm, stride);
    __syncthreads();
    const int r = threadIdx.x;
    if (r < cr) {
      const float* row = &sm[r * stride];
      float4* dst = reinterpret_cast<float4*>(U + (long long)(t.row0 + r0 + r) * rcap);
      for (int g0 = 0; g0 < c4; g0 += 2) {
        float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
        const bool two = (g0 + 1) < c4;
        for (int c = 0; c < n; ++c) {
          const float x = row[c];
          const float4 v0 = *reinterpret_cast<const float4*>(&vs[c * RCAP_MAX + 4 * g0]);
          a0.x = fmaf(x, v0.x, a0.x); a0.y = fmaf(x, v0.y, a0.y);
          a0.z = fmaf(x, v0.z, a0.z); a0.w = fmaf(x, v0.w, a0.w);
          if (two) {
            const float4 v1 = *reinterpret_cast<const float4*>(&vs[c * RCAP_MAX + 4 * g0 + 4]);
            a1.x = fmaf(x, v1.x, a1.x); a1.y = fmaf(x, v1.y, a1.y);
            a1.z = fmaf(x, v1.z, a1.z); a1.w = fmaf(x, v1.w, a1.w);
          }
        }
        st_na_f4(dst + g0, a0);
        if (two) st_na_f4(dst + g0 + 1, a1);
      }
    }
  }

  // ---- completion: last CTA publishes flag[worker] = step ------------------------------
  if (signal) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      const unsigned int old = atomicAdd(&ctrl->done_encode, 1u);
      if (old == gridDim.x - 1) {
        ctrl->done_encode = 0;
        __threadfence_system();
        st_release_sys(push_flag_peer + worker_index, ctrl->step);
      }
    }
  }
}

// flag-only publication (configs with no tall-skinny layer, or dense-only pushes)
__global__ void signal_push_kernel(int* push_flag_peer, const Ctrl* ctrl, int worker_index) {
  if (threadIdx.x == 0) {
    __threadfence_system();
    st_release_sys(push_flag_peer + worker_index, ctrl->step);
  }
}

// ----------------------------------------------------------------------------
// host launchers (plain C ABI; bindings.cpp wraps them for torch)
// ----------------------------------------------------------------------------
extern "C" {

void atomo_launch_gram(const float* grad, const void* layers, const void* tiles, int ntiles, float* gpart,
                       cudaStream_t stream) {
  if (ntiles <= 0) return;
  gram_kernel<<<ntiles, GRAM_THREADS, 0, stream>>>(grad, (const LayerDesc*)layers, (const TileDesc*)tiles, gpart);
}

void atomo_launch_eig_sample(const void* layers, const int* ts_layers, int n_ts, const float* gpart, float* vsel,
                             int* selcount, float* sigma_out, float* ps_arena_peer, long long arena_floats,
                             const void* ctrl, const float* ext_uniforms, int rank, int random_sample,
                             int waterfill, int systematic, int worker_index, int threads, cudaStream_t stream) {
  if (n_ts <= 0) return;
  if (threads < 64) threads = EIG_THREADS;
  if (threads > 1024) threads = 1024;
  EncodeCfg cfg{rank, random_sample, waterfill, systematic, worker_index, ext_uniforms != nullptr};
  eig_sample_kernel<<<n_ts, threads, 0, stream>>>((const LayerDesc*)layers, ts_layers, gpart, vsel, selcount,
                                                        sigma_out, ps_arena_peer, arena_floats, (const Ctrl*)ctrl,
                                                        ext_uniforms, cfg);
}

void atomo_launch_project_push(const float* grad, const void* layers, const void* tiles, int ntiles,
                               const float* vsel, const int* selcount, float* ps_arena_peer,
                               long long arena_floats, int* push_flag_peer, void* ctrl, int worker_index,
                               int signal, cudaStream_t stream) {
  if (ntiles <= 0) {
    if (signal) signal_push_kernel<<<1, 32, 0, stream>>>(push_flag_peer, (const Ctrl*)ctrl, worker_index);
    return;
  }
  project_push_kernel<<<ntiles, PROJ_THREADS, 0, stream>>>(grad, (const LayerDesc*)layers, (const TileDesc*)tiles,
                                                            vsel, selcount, ps_arena_peer, arena_floats,
                                                            push_flag_peer, (Ctrl*)ctrl, worker_index, signal);
}

void atomo_launch_signal_push(int* push_flag_peer, const void* ctrl, int worker_index, cudaStream_t stream) {
  signal_push_kernel<<<1, 32, 0, stream>>>(push_flag_peer, (const Ctrl*)ctrl, worker_index);
}

}  // extern "C"
}  // namespace atomo
