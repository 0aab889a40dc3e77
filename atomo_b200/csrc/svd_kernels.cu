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
//                      Philox Bernoulli / systematic sampling (spectral_sample.cuh,
//                      shared with the bf16 engine's v2_encode_kernel);
//                      header, s_a = sigma_a/p_a and V rows -> PS slot (peer store)
//   project_push     : U[:,a] = A v_a / sigma_a            (pass 2, L2-resident)
//                      float4 peer stores of U into the PS slot; the last CTA
//                      publishes the step-stamped flag with st.release.sys.
//
// Because V is a complete orthonormal basis of the skinny dimension,
// sum_i (A v_i) v_i^T == A exactly, so the estimator is unbiased even when the
// fp32 Gram/Jacobi eigenvectors are only approximately the singular vectors.
#include "spectral_sample.cuh"

namespace atomo {

constexpr int GRAM_THREADS = 256;
constexpr int GRAM_CHUNK = 64;   // rows staged per iteration
constexpr int EIG_THREADS = 256;
constexpr int PROJ_THREADS = 128;

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
};

__global__ void __launch_bounds__(1024)
eig_sample_kernel(const LayerDesc* __restrict__ layers, const int* __restrict__ ts_layers,
                  const float* __restrict__ gpart, float* __restrict__ vsel, int* __restrict__ selcount,
                  float* __restrict__ sigma_out, float* ps_arena_peer, long long arena_floats, const Ctrl* ctrl,
                  const float* __restrict__ ext_uniforms, EncodeCfg cfg) {
  __shared__ float G[TS_MAX_COLS * SPECTRAL_PITCH];
  __shared__ float V[TS_MAX_COLS * SPECTRAL_PITCH];

  const int layer_id = ts_layers[blockIdx.x];
  const LayerDesc L = layers[layer_id];
  const int n = L.cols;
  const int tid = threadIdx.x;
  const int step = ctrl->step;

  // ---- G = sum of tile partials (padded to an even size with a zero row/col); V = I ----------
  const int ne = n + (n & 1);
  for (int e = tid; e < ne * ne; e += blockDim.x) {
    const int i = e / ne, j = e - i * ne;
    float s = 0.f;
    if (i < n && j < n) {
      const float* gp = gpart + L.gpart_off + i * n + j;
      for (int t = 0; t < L.ntiles; ++t) s += gp[(long long)t * n * n];
    }
    G[i * SPECTRAL_PITCH + j] = s;
    V[i * SPECTRAL_PITCH + j] = (i == j) ? 1.f : 0.f;
  }
  __syncthreads();
  // symmetrize (partials are accumulated in different orders for (i,j)/(j,i))
  for (int e = tid; e < n * n; e += blockDim.x) {
    int i = e / n, j = e - i * n;
    if (i < j) {
      float v = 0.5f * (G[i * SPECTRAL_PITCH + j] + G[j * SPECTRAL_PITCH + i]);
      G[i * SPECTRAL_PITCH + j] = v;
      G[j * SPECTRAL_PITCH + i] = v;
    }
  }
  __syncthreads();

  // ---- Jacobi, sampling (an empty draw is always redrawn), vsel[blockIdx.x] = V[:, sel] / sigma ------------
  const int rcap = L.rcap;
  const SampleCfg scfg{(float)cfg.rank, rcap, cfg.random_sample, cfg.waterfill, cfg.systematic, 1,
                       ext_uniforms, &ctrl->seed, layer_id,
                       ((uint32_t)cfg.worker_index << 24) ^ (uint32_t)step};
  const Spectrum sp = eig_sample(G, V, n, false, 0, scfg, blockIdx.x, vsel, nullptr, 0, false);
  const int count = sp.count;

  // ---- publish: selection count, sigma, and the PS slot header / s / V ----------------------------------
  if (tid == 0) selcount[blockIdx.x] = count;
  if (sigma_out != nullptr && tid < n) sigma_out[(long long)blockIdx.x * TS_MAX_COLS + tid] = sp.sig[sp.order[tid]];

  float* slot = ps_arena_peer + (long long)cfg.worker_index * arena_floats + L.slot_off;
  if (tid < rcap) slot[slot_s_off() + tid] = (tid < count) ? sp.sig[sp.sel[tid]] * sp.selscale[tid] : 0.f;
  float* vout = slot + slot_v_off(rcap);
  for (int e = tid; e < rcap * n; e += blockDim.x) {
    const int a = e / n, c = e - a * n;
    vout[e] = (a < count) ? V[c * SPECTRAL_PITCH + sp.sel[a]] : 0.f;
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
  EncodeCfg cfg{rank, random_sample, waterfill, systematic, worker_index};
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
