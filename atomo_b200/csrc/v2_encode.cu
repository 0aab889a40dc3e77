// Worker side of the overlapped engine: spectral-ATOMO encode of ONE backward group, fused with the push
// into the parameter-server owners' HBM over NVLink (sm_90a).
//
// Reference pipeline per tensor (SURVEY.md 2.5 K1): D2H copy -> numpy LAPACK SVD (codings/svd.py:95) ->
// Python Bernoulli loop (svd.py:49-67) -> pickle -> MPI isend (distributed_worker.py:313-335), strictly after
// the whole backward.  Here, per group of layers and while backward is still running on the main stream:
//
//   v2_encode_kernel   one CTA per tile of bf16 gradient, read where cuDNN wrote it ([O][K][I] slabs):
//                      TMA bulk copies (cp.async.bulk + mbarrier) into shared memory, Gram matrix of the
//                      tile in 4x4 register blocks (fp32 accumulate), partial written out; the LAST tile of a unit sums the partials and runs
//                      the Jacobi eigensolver + atom sampling in the same launch (no separate eig kernel),
//                      then stores header / s / V into every owner's slot through peer pointers.
//   v2_project_kernel  U = A V / sigma for the sampled atoms (second pass, L2 resident), float4 peer stores of
//                      each row into the arena of the PS owner of that row's tile; the last CTA of the group
//                      publishes flag[group][worker] = step on every owner with st.release.sys.  With error
//                      feedback (v2_feedback.cu) each row also adds A - U diag(s) V^T, the part of the coded input
//                      the owner does not reconstruct, to the worker's fp32 residual.
#include "spectral_sample.cuh"
#include "v2_common.cuh"

namespace atomo {
namespace v2 {

constexpr int ENC_THREADS = 256;
constexpr int ENC_HDR = 128;
constexpr int ENC_TILE_BYTES = 36 * 1024;       // tile buffer; reused for G / V (2 x 64 x 65 floats) in the eig phase
constexpr int ENC_RED_BYTES = 64 * 64 * 4;
constexpr int ENC_SMEM = ENC_HDR + ENC_TILE_BYTES + ENC_RED_BYTES;

struct EncCfg {
  int random_sample;
  int waterfill;
  int systematic;
  int worker;
  int resample_empty;   // 1 = the reference's rule (svd.py:65-66: redraw when nothing was selected; biased by
                        // 1/(1-P(empty)), ~e^-budget), 0 = send zero atoms (exactly unbiased; default)
};

struct EncArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  const long long* gptr;       // gradient base pointers (bf16), one per weight tensor
  float* gpart;
  unsigned int* unit_counters;
  float* vsel;                 // [n_coded][64][32]   V[:, sel] / sigma
  int* selcount;
  float* sigma_out;            // optional [n_coded][64]
  float* const* arena_peer;    // [n_owners] arena base inside each owner
  int n_owners;
  long long arena_floats;
  __nv_bfloat16* stage;        // local staging region of the dense bf16 weights
  const Ctrl2* ctrl;
  const float* ext_uniforms;   // tests: [n_coded][64] uniforms replacing Philox on the first attempt
  float* vprev;                // [n_coded][64*64] eigenbasis of the previous step (warm start), or nullptr
  int max_sweeps;              // Jacobi sweep cap (any complete orthonormal basis keeps the estimator unbiased)
  int flags;                   // bit 0: load tiles with plain loads instead of TMA bulk copies
  long long* tstats;           // device-side phase accounting (see runtime/shadow_engine.py: phase_stats)
  int group;
  EncCfg cfg;
};

// ------------------------------------------------------------------------------------------------------
// Gram of a SLAB tile.  Z[c][p] (c = b*K + k, p = channel pair) = X[k][2p + b]; G = Z Z^T.
//
// CUDA-core FFMA: the Gram is 0.1 GFLOP per step against 21 MB of gradient, i.e. bandwidth bound, and this
// kernel shares SMs with cuDNN's backward kernels (it runs on a side stream during backward), so it keeps its
// register / shared-memory footprint small (63 registers, 4 CTAs per SM) instead of chasing tensor-core peak.
//
// Thread layout: internal column order c' = 2k + b, so that 4 consecutive columns are the two halves of two
// words.  A thread owns one 4x4 block (bi <= bj) of G for a subset of the rows; per row it loads 4 words and
// issues 16 FMAs.  Row groups are summed through the (then idle) tile buffer, without shared atomics.
// ------------------------------------------------------------------------------------------------------
__device__ void slab_gram(const uint32_t* sm, int K, int I, int ns, float* red, int npad, int n, float* stage) {
  const int pitch = slab_pitch_words(I), half = I >> 1;
  const int nb = (2 * K + 3) >> 2;             // 4-column blocks in c' order
  const int nbp = nb * (nb + 1) / 2;
  const int RG = max(1, (int)blockDim.x / nbp);
  const int pb = threadIdx.x % nbp, grp = threadIdx.x / nbp;
  int bi = 0, rem = pb;
  while (rem >= nb - bi) { rem -= nb - bi; ++bi; }
  const int bj = bi + rem;
  const bool active = grp < RG;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  if (active) {
    const int ki0 = min(2 * bi, K - 1), ki1 = min(2 * bi + 1, K - 1);   // clamped taps: padding columns are dropped below
    const int kj0 = min(2 * bj, K - 1), kj1 = min(2 * bj + 1, K - 1);
    int s = grp / half, ri = grp - s * half;
    const int ds = RG / half, dri = RG - ds * half;
    while (s < ns) {
      const uint32_t* base = sm + (size_t)(s * K) * pitch + ri;
      const uint32_t wi0 = base[ki0 * pitch], wi1 = base[ki1 * pitch];
      const uint32_t wj0 = base[kj0 * pitch], wj1 = base[kj1 * pitch];
      const float ai[4] = {bf16_lo(wi0), bf16_hi(wi0), bf16_lo(wi1), bf16_hi(wi1)};
      const float aj[4] = {bf16_lo(wj0), bf16_hi(wj0), bf16_lo(wj1), bf16_hi(wj1)};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ai[i], aj[j], acc[i][j]);
      s += ds; ri += dri;
      if (ri >= half) { ri -= half; ++s; }
    }
  }
  __syncthreads();   // `stage` aliases the tile buffer: every thread is done reading the tile
  if (active) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) stage[(grp * 16 + i * 4 + j) * nbp + pb] = acc[i][j];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 16 * nbp; e += blockDim.x) {
    const int v = e / nbp, q = e - v * nbp;
    float sum = 0.f;
    for (int g = 0; g < RG; ++g) sum += stage[(g * 16 + v) * nbp + q];
    int qi = 0, qr = q;
    while (qr >= nb - qi) { qr -= nb - qi; ++qi; }
    const int qj = qi + qr;
    const int ci_ = 4 * qi + (v >> 2), cj_ = 4 * qj + (v & 3);      // c' indices
    const int k_i = ci_ >> 1, k_j = cj_ >> 1;
    if (k_i < K && k_j < K) {
      const int ci = (ci_ & 1) * K + k_i, cj = (cj_ & 1) * K + k_j;  // c = b*K + k
      if (qi != qj || ci_ <= cj_) red[min(ci, cj) * npad + max(ci, cj)] = sum;
    }
  }
}

// MAT tile: rows [r0, r0+nr) of a strided bf16 matrix staged as fp32 [nr][npad], 4x4 register blocks (FFMA)
__device__ void mat_gram(const __nv_bfloat16* gb, const Unit2& u, int r0, int nr, float* smf, float* red, int npad,
                         int n) {
  const int tid = threadIdx.x;
  if (u.cs == 1) {
    for (int e = tid; e < nr * n; e += blockDim.x) {
      const int r = e / n, c = e - r * n;
      smf[r * npad + c] = __bfloat162float(gb[(long long)(r0 + r) * u.rs + c]);
    }
  } else {
    for (int e = tid; e < nr * n; e += blockDim.x) {
      const int c = e / nr, r = e - c * nr;
      smf[r * npad + c] = __bfloat162float(gb[(long long)(r0 + r) * u.rs + (long long)c * u.cs]);
    }
  }
  if (npad > n)
    for (int e = tid; e < nr * (npad - n); e += blockDim.x) {
      const int r = e / (npad - n), c = n + e - r * (npad - n);
      smf[r * npad + c] = 0.f;
    }
  __syncthreads();
  const int nb = npad >> 2, NB = nb * nb;
  // RG row groups; their partial blocks are added into `red` one group after the other (not with atomics), so the
  // Gram matrix has the same bits on every run
  const int RG = min(16, max(1, (int)blockDim.x / NB));
  const int blk = tid % NB, grp = tid / NB;
  const int bi = blk / nb, bj = blk - bi * nb;
  const bool active = grp < RG && bi <= bj;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  if (active) {
    for (int r = grp; r < nr; r += RG) {
      const float4 a = *reinterpret_cast<const float4*>(&smf[r * npad + 4 * bi]);
      const float4 b = *reinterpret_cast<const float4*>(&smf[r * npad + 4 * bj]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
  for (int g = 0; g < RG; ++g) {
    if (active && grp == g) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int r = 4 * bi + i, c = 4 * bj + j;
          if (r <= c && c < n) red[r * npad + c] += acc[i][j];
        }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------------
// Eigen-decomposition of the unit's Gram + atom sampling (spectral_sample.cuh).  Runs in the LAST encode CTA of the
// unit; G / V live in the tile buffer.
// ------------------------------------------------------------------------------------------------------
__device__ void eig_sample_unit(const EncArgs& a, const Unit2& u, int unit_id, float* G, float* V, float* Tbuf) {
  const int n = u.cols, tid = threadIdx.x, nthr = blockDim.x;
  const int step = a.ctrl->step;
  const int ts = u.ts_index;
  const int ne = n + (n & 1);
  // Warm start: the right-singular basis of a layer's gradient drifts slowly from step to step, so Jacobi starts
  // from last step's basis V0 (G0 = V0^T G V0 is already nearly diagonal) and needs 1-2 sweeps instead of 6-10.
  // The basis is reset to the identity every 256 steps so rounding drift of V's orthonormality cannot build up.
  float* vp = a.vprev != nullptr ? a.vprev + (long long)ts * V2_MAX_COLS * V2_MAX_COLS : nullptr;
  const bool warm = vp != nullptr && (step & 255) != 0;
  for (int e = tid; e < ne * ne; e += nthr) {
    const int i = e / ne, j = e - i * ne;
    float s = 0.f;
    if (i < n && j < n) {
      const float* gp = a.gpart + u.gpart_off + i * n + j;
      for (int t = 0; t < u.n_enc; ++t) s += __ldcg(gp + (long long)t * n * n);
    }
    G[i * SPECTRAL_PITCH + j] = s;
    float v0 = (i == j) ? 1.f : 0.f;
    if (warm && i < n && j < n) v0 = vp[i * n + j];
    V[i * SPECTRAL_PITCH + j] = v0;
  }
  if (warm) {
    float* T = Tbuf;   // n x n scratch (the Gram reduction buffer of the tile phase)
    __syncthreads();
    for (int e = tid; e < n * n; e += nthr) {       // T = G V0
      const int i = e / n, j = e - i * n;
      float acc = 0.f;
      for (int k = 0; k < n; ++k) acc = fmaf(G[i * SPECTRAL_PITCH + k], V[k * SPECTRAL_PITCH + j], acc);
      T[e] = acc;
    }
    __syncthreads();
    for (int e = tid; e < n * n; e += nthr) {       // G0 = V0^T T, symmetrized
      const int i = e / n, j = e - i * n;
      if (i <= j) {
        float x = 0.f, y = 0.f;
        for (int k = 0; k < n; ++k) {
          x = fmaf(V[k * SPECTRAL_PITCH + i], T[k * n + j], x);
          y = fmaf(V[k * SPECTRAL_PITCH + j], T[k * n + i], y);
        }
        const float v = 0.5f * (x + y);
        G[i * SPECTRAL_PITCH + j] = v;
        G[j * SPECTRAL_PITCH + i] = v;
      }
    }
  }
  __syncthreads();
  // warm: a.max_sweeps refinement sweeps track the slowly drifting basis; cold (first step / periodic reset): full solve.
  // Stores vsel[ts], the projection basis of v2_project_kernel.
  const SampleCfg cfg{u.budget, u.rcap, a.cfg.random_sample, a.cfg.waterfill, a.cfg.systematic, a.cfg.resample_empty,
                      a.ext_uniforms, &a.ctrl->seed, unit_id, ((uint32_t)a.cfg.worker << 24) ^ (uint32_t)step};
  const Spectrum sp = eig_sample(G, V, n, warm, a.max_sweeps, cfg, ts, a.vsel, const_cast<int*>(&a.ctrl->error),
                                 ERR2_NONFINITE, true);
  const int count = sp.count, rcap = u.rcap;

  // ---- publish: selection count, next step's warm start, and header / s / V into every owner's slot ----
  if (tid == 0) a.selcount[ts] = count;
  if (vp != nullptr)
    for (int e = tid; e < n * n; e += nthr) vp[e] = V[(e / n) * SPECTRAL_PITCH + (e % n)];
  if (a.sigma_out != nullptr && tid < n) a.sigma_out[(long long)ts * V2_MAX_COLS + tid] = sp.sig[sp.order[tid]];
  // header / s / V go to every owner's slot.  Only warp 0 stores (and fences): a system-scope fence per thread
  // of the CTA costs microseconds, one per lane of a single warp is one instruction.
  if (tid < 32) {
    for (int o = 0; o < a.n_owners; ++o) {
      float* slot = a.arena_peer[o] + (long long)a.cfg.worker * a.arena_floats + u.slot_off;
      for (int x = tid; x < rcap; x += 32) slot[4 + x] = (x < count) ? sp.sig[sp.sel[x]] * sp.selscale[x] : 0.f;
      float* vout = slot + 4 + rcap;
      for (int e = tid; e < rcap * n; e += 32) {
        const int x = e / n, c = e - x * n;
        vout[e] = (x < count) ? V[c * SPECTRAL_PITCH + sp.sel[x]] : 0.f;
      }
      if (tid == 0) {
        int* hdr = reinterpret_cast<int*>(slot);
        hdr[0] = count; hdr[1] = step; hdr[2] = n; hdr[3] = u.rows;
      }
    }
    __threadfence_system();
  }
}

extern __shared__ __align__(128) unsigned char enc_smem[];

__global__ void __launch_bounds__(ENC_THREADS) v2_encode_kernel(const EncArgs a) {
  uint64_t* mbar = reinterpret_cast<uint64_t*>(enc_smem);
  uint32_t* tile = reinterpret_cast<uint32_t*>(enc_smem + ENC_HDR);
  float* red = reinterpret_cast<float*>(enc_smem + ENC_HDR + ENC_TILE_BYTES);
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x;
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();

  if (u.kind == KIND_DENSE16) {
    // staging copy of a dense bf16 gradient into the symmetric heap (the PS owners pull it from there)
    __nv_bfloat16* dst = a.stage + u.rs + t.a;
    const __nv_bfloat16* src = gb + t.a;
    if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
      const int nv = t.b >> 3;
      for (int i = tid; i < nv; i += blockDim.x)
        reinterpret_cast<uint4*>(dst)[i] = __ldg(reinterpret_cast<const uint4*>(src) + i);
      for (int i = (nv << 3) + tid; i < t.b; i += blockDim.x) dst[i] = src[i];
    } else {
      for (int i = tid; i < t.b; i += blockDim.x) dst[i] = src[i];
    }
    return;
  }

  const int n = u.cols;
  const int npad = (n + 3) & ~3;
  for (int i = tid; i < npad * npad; i += blockDim.x) red[i] = 0.f;
  if (u.kind == KIND_SLAB) {
    if (tid == 0) { mbar_init(mbar, 1); mbar_fence_init(); }
    __syncthreads();
    if (a.flags & 1) {
      load_slab_tile_ldg(gb + (long long)t.a * u.K * u.I, u.K, u.I, t.b, tile);
      __syncthreads();
    } else {
      load_slab_tile(gb + (long long)t.a * u.K * u.I, u.K, u.I, t.b, tile, mbar);
      mbar_wait(mbar, 0);
    }
    slab_gram(tile, u.K, u.I, t.b, red, npad, n, reinterpret_cast<float*>(tile));
  } else {
    __syncthreads();
    mat_gram(gb, u, t.a, t.b, reinterpret_cast<float*>(tile), red, npad, n);
  }
  __syncthreads();
  // partial Gram of this tile (full symmetric n x n)
  {
    const int local_tile = t.owner;   // encode tiles: Tile2::owner holds the tile's index inside its unit
    float* o2 = a.gpart + u.gpart_off + (long long)local_tile * n * n;
    for (int e = tid; e < n * n; e += blockDim.x) {
      const int i = e / n, j = e - i * n;
      o2[e] = i <= j ? red[i * npad + j] : red[j * npad + i];
    }
  }
  // ---- last tile of the unit: eigen-decomposition + sampling in the same launch -----------------
  __threadfence();   // every thread publishes its own slice of the partial before the CTA is counted
  __syncthreads();
  if (tid == 0) {
    const unsigned int old = atomicAdd(&a.unit_counters[u.ts_index], 1u);
    s_last = (old == (unsigned int)u.n_enc - 1u) ? 1 : 0;
    if (s_last) a.unit_counters[u.ts_index] = 0;
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    float* G = reinterpret_cast<float*>(tile);
    float* V = G + V2_MAX_COLS * SPECTRAL_PITCH;
    eig_sample_unit(a, u, t.unit, G, V, red);
  }
}

// ------------------------------------------------------------------------------------------------------
// pass 2: U rows -> owner arenas; last CTA of the group raises flag[group][worker] on every owner
// ------------------------------------------------------------------------------------------------------
struct ProjArgs {
  const Unit2* units;
  const Tile2* tiles;
  const long long* gptr;
  const float* vsel;
  const int* selcount;
  float* const* arena_peer;
  int* const* sig_peer;        // [n_owners] signal region base of each owner
  int n_owners;
  long long arena_floats;
  int worker;
  int group;
  Ctrl2* ctrl;
  unsigned int* group_counter;
  int flags;
  long long* tstats;
  int final_group;
  int timed;          // 1 when an encode launch of this group stamped its start time
};

constexpr int PROJ_SMEM = ENC_HDR + ENC_TILE_BYTES + V2_MAX_COLS * V2_RCAP_MAX * 4;
// error feedback adds s_x V[x][c] (as the owner forms it) and every thread's U row
constexpr int PROJ_EF_SMEM = PROJ_SMEM + V2_MAX_COLS * V2_RCAP_MAX * 4 + V2_RCAP_MAX * ENC_THREADS * 4;

// Error feedback: U[x] s_x V[x][c] summed over the atoms in atom order with fmaf, which is the order and rounding of
// the owner's reconstruction (v2_ps_kernel) for one worker
__device__ __forceinline__ float ef_recon(const float* ust, const float* svc, int count) {
  float acc = 0.f;
  for (int x = 0; x < count; ++x) acc = fmaf(ust[x * ENC_THREADS], svc[x], acc);
  return acc;
}

// QSVD: quantize one float4 of a U row to 4 x int8 with unbiased stochastic rounding against the row scale
__device__ __forceinline__ int quant4_i8(const float4 v, float inv_scale127, const uint32_t (&rnd)[4]) {
  const float x[4] = {v.x, v.y, v.z, v.w};
  int packed = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float t = x[j] * inv_scale127;                       // in [-127, 127]
    const float fl = floorf(t);
    int q = (int)fl + ((Philox::to_uniform(rnd[j]) < (t - fl)) ? 1 : 0);
    q = max(-127, min(127, q));
    packed |= (q & 0xff) << (8 * j);
  }
  return packed;
}

// EF (v2_project_ef_kernel): `residual` is the fp32 residual indexed like wshadow, `ef_owner` the owner whose copy of
// this worker's slot (s, V) the epilogue reads (a local one if any)
template <bool EF>
__device__ __forceinline__ void project(const ProjArgs& a, float* residual, int ef_owner) {
  uint64_t* mbar = reinterpret_cast<uint64_t*>(enc_smem);
  uint32_t* tile = reinterpret_cast<uint32_t*>(enc_smem + ENC_HDR);
  float* vs = reinterpret_cast<float*>(enc_smem + ENC_HDR + ENC_TILE_BYTES);
  float* sv = vs + V2_MAX_COLS * V2_RCAP_MAX;          // error feedback only: [col][atom] s_x V[x][col]
  float* ust = sv + V2_MAX_COLS * V2_RCAP_MAX;         // error feedback only: [atom][thread] U row of the thread
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x;
  const bool ef = EF && u.ubits != 8;

  if (u.kind == KIND_SLAB || u.kind == KIND_MAT) {
    const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
    const int n = u.cols, rcap = u.rcap;
    const int count = a.selcount[u.ts_index];
    const int c4 = (count + 3) >> 2;
    if (u.kind == KIND_SLAB) {
      if (tid == 0) { mbar_init(mbar, 1); mbar_fence_init(); }
      __syncthreads();
      if (a.flags & 1) load_slab_tile_ldg(gb + (long long)t.a * u.K * u.I, u.K, u.I, t.b, tile);
      else load_slab_tile(gb + (long long)t.a * u.K * u.I, u.K, u.I, t.b, tile, mbar);
    }
    const float* vsrc = a.vsel + (long long)u.ts_index * V2_MAX_COLS * V2_RCAP_MAX;
    for (int e = tid; e < n * V2_RCAP_MAX; e += blockDim.x) vs[e] = vsrc[e];
    if (ef) {       // the slot's s and V, as the encode launch stored them
      const float* slot = a.arena_peer[ef_owner] + (long long)a.worker * a.arena_floats + u.slot_off;
      for (int e = tid; e < n * V2_RCAP_MAX; e += blockDim.x) {
        const int c = e / V2_RCAP_MAX, x = e - c * V2_RCAP_MAX;
        sv[e] = (x < count) ? slot[4 + x] * slot[4 + rcap + (long long)x * n + c] : 0.f;
      }
    }
    __syncthreads();
    const long long uoff = (long long)a.worker * a.arena_floats + u.slot_off + slot2_u_off(rcap, n);
    if (u.kind == KIND_SLAB) {
      if (!(a.flags & 1)) mbar_wait(mbar, 0);
      const int K = u.K, half = u.I >> 1, pitch = slab_pitch_words(u.I);
      const int nrows = t.b * half;
      for (int rl = tid; rl < nrows; rl += blockDim.x) {
        const int s = rl / half, ri = rl - s * half;
        const long long r = (long long)(t.a + s) * half + ri;
        const int owner = (u.own0 + (int)(r / u.ps_rows)) % a.n_owners;
        float4* dst = reinterpret_cast<float4*>(a.arena_peer[owner] + uoff + r * rcap);
        const uint32_t* col = tile + (size_t)(s * K) * pitch + ri;
        float rowmax = 0.f;          // QSVD: first pass finds max |u| of the row, second pass quantizes
        for (int pass = (u.ubits == 8 ? 0 : 1); pass < 2; ++pass)
        for (int g0 = 0; g0 < c4; g0 += 2) {
          float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
          const bool two = (g0 + 1) < c4;
          for (int k = 0; k < K; ++k) {
            const uint32_t w = col[k * pitch];
            const float x0 = bf16_lo(w), x1 = bf16_hi(w);
            const float4 v0 = *reinterpret_cast<const float4*>(&vs[k * V2_RCAP_MAX + 4 * g0]);
            const float4 v1 = *reinterpret_cast<const float4*>(&vs[(K + k) * V2_RCAP_MAX + 4 * g0]);
            a0.x = fmaf(x0, v0.x, a0.x); a0.y = fmaf(x0, v0.y, a0.y);
            a0.z = fmaf(x0, v0.z, a0.z); a0.w = fmaf(x0, v0.w, a0.w);
            a0.x = fmaf(x1, v1.x, a0.x); a0.y = fmaf(x1, v1.y, a0.y);
            a0.z = fmaf(x1, v1.z, a0.z); a0.w = fmaf(x1, v1.w, a0.w);
            if (two) {
              const float4 w0 = *reinterpret_cast<const float4*>(&vs[k * V2_RCAP_MAX + 4 * g0 + 4]);
              const float4 w1 = *reinterpret_cast<const float4*>(&vs[(K + k) * V2_RCAP_MAX + 4 * g0 + 4]);
              a1.x = fmaf(x0, w0.x, a1.x); a1.y = fmaf(x0, w0.y, a1.y);
              a1.z = fmaf(x0, w0.z, a1.z); a1.w = fmaf(x0, w0.w, a1.w);
              a1.x = fmaf(x1, w1.x, a1.x); a1.y = fmaf(x1, w1.y, a1.y);
              a1.z = fmaf(x1, w1.z, a1.z); a1.w = fmaf(x1, w1.w, a1.w);
            }
          }
          if (u.ubits != 8) {
            st_na_f4(dst + g0, a0);
            if (two) st_na_f4(dst + g0 + 1, a1);
            if (ef) {
              float* us = ust + 4 * g0 * ENC_THREADS + tid;
              us[0] = a0.x; us[ENC_THREADS] = a0.y; us[2 * ENC_THREADS] = a0.z; us[3 * ENC_THREADS] = a0.w;
              if (two) {
                us[4 * ENC_THREADS] = a1.x; us[5 * ENC_THREADS] = a1.y;
                us[6 * ENC_THREADS] = a1.z; us[7 * ENC_THREADS] = a1.w;
              }
            }
          } else if (pass == 0) {
            rowmax = fmaxf(rowmax, fmaxf(fmaxf(fabsf(a0.x), fabsf(a0.y)), fmaxf(fabsf(a0.z), fabsf(a0.w))));
            if (two) rowmax = fmaxf(rowmax, fmaxf(fmaxf(fabsf(a1.x), fabsf(a1.y)), fmaxf(fabsf(a1.z), fabsf(a1.w))));
          } else {
            float* sbase = a.arena_peer[owner] + (long long)a.worker * a.arena_floats + u.slot_off;
            int* q8 = reinterpret_cast<int*>(sbase + slot2_u_off(rcap, n)) + (r * rcap >> 2);
            const float inv = rowmax > 0.f ? 127.f / rowmax : 0.f;
            uint32_t rnd[4];
            Philox::gen(a.ctrl->seed ^ 0x51ed270b1ULL, (uint32_t)r, (uint32_t)g0, (uint32_t)t.unit,
                        ((uint32_t)a.worker << 24) ^ (uint32_t)a.ctrl->step, rnd);
            q8[g0] = quant4_i8(a0, inv, rnd);
            if (two) {
              Philox::gen(a.ctrl->seed ^ 0x51ed270b1ULL, (uint32_t)r, (uint32_t)(g0 + 1), (uint32_t)t.unit,
                          ((uint32_t)a.worker << 24) ^ (uint32_t)a.ctrl->step, rnd);
              q8[g0 + 1] = quant4_i8(a1, inv, rnd);
            }
            if (g0 == 0) sbase[slot2_scale_off(u.rows, rcap, n) + r] = rowmax;
          }
        }
        if (ef) {     // e += A - U diag(s) V^T on the row's 2K elements (s, k, 2ri + b); float2 aligned (I % 16 == 0)
          float* er = residual + u.w_off + (long long)(t.a + s) * K * u.I + 2 * ri;
          for (int k = 0; k < K; ++k) {
            const uint32_t w = col[k * pitch];
            float2* p = reinterpret_cast<float2*>(er + (long long)k * u.I);
            float2 e = *p;
            e.x += bf16_lo(w) - ef_recon(ust + tid, sv + k * V2_RCAP_MAX, count);
            e.y += bf16_hi(w) - ef_recon(ust + tid, sv + (K + k) * V2_RCAP_MAX, count);
            *p = e;
          }
        }
      }
    } else {
      for (int rl = tid; rl < t.b; rl += blockDim.x) {
        const long long r = t.a + rl;
        const int owner = (u.own0 + (int)(r / u.ps_rows)) % a.n_owners;
        float4* dst = reinterpret_cast<float4*>(a.arena_peer[owner] + uoff + r * rcap);
        const __nv_bfloat16* row = gb + r * u.rs;
        float rowmax = 0.f;
        for (int pass = (u.ubits == 8 ? 0 : 1); pass < 2; ++pass)
        for (int g0 = 0; g0 < c4; g0 += 2) {
          float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
          const bool two = (g0 + 1) < c4;
          for (int c = 0; c < n; ++c) {
            const float x = __bfloat162float(row[(long long)c * u.cs]);
            const float4 v0 = *reinterpret_cast<const float4*>(&vs[c * V2_RCAP_MAX + 4 * g0]);
            a0.x = fmaf(x, v0.x, a0.x); a0.y = fmaf(x, v0.y, a0.y);
            a0.z = fmaf(x, v0.z, a0.z); a0.w = fmaf(x, v0.w, a0.w);
            if (two) {
              const float4 v1 = *reinterpret_cast<const float4*>(&vs[c * V2_RCAP_MAX + 4 * g0 + 4]);
              a1.x = fmaf(x, v1.x, a1.x); a1.y = fmaf(x, v1.y, a1.y);
              a1.z = fmaf(x, v1.z, a1.z); a1.w = fmaf(x, v1.w, a1.w);
            }
          }
          if (u.ubits != 8) {
            st_na_f4(dst + g0, a0);
            if (two) st_na_f4(dst + g0 + 1, a1);
            if (ef) {
              float* us = ust + 4 * g0 * ENC_THREADS + tid;
              us[0] = a0.x; us[ENC_THREADS] = a0.y; us[2 * ENC_THREADS] = a0.z; us[3 * ENC_THREADS] = a0.w;
              if (two) {
                us[4 * ENC_THREADS] = a1.x; us[5 * ENC_THREADS] = a1.y;
                us[6 * ENC_THREADS] = a1.z; us[7 * ENC_THREADS] = a1.w;
              }
            }
          } else if (pass == 0) {
            rowmax = fmaxf(rowmax, fmaxf(fmaxf(fabsf(a0.x), fabsf(a0.y)), fmaxf(fabsf(a0.z), fabsf(a0.w))));
            if (two) rowmax = fmaxf(rowmax, fmaxf(fmaxf(fabsf(a1.x), fabsf(a1.y)), fmaxf(fabsf(a1.z), fabsf(a1.w))));
          } else {
            float* sbase = a.arena_peer[owner] + (long long)a.worker * a.arena_floats + u.slot_off;
            int* q8 = reinterpret_cast<int*>(sbase + slot2_u_off(rcap, n)) + (r * rcap >> 2);
            const float inv = rowmax > 0.f ? 127.f / rowmax : 0.f;
            uint32_t rnd[4];
            Philox::gen(a.ctrl->seed ^ 0x51ed270b1ULL, (uint32_t)r, (uint32_t)g0, (uint32_t)t.unit,
                        ((uint32_t)a.worker << 24) ^ (uint32_t)a.ctrl->step, rnd);
            q8[g0] = quant4_i8(a0, inv, rnd);
            if (two) {
              Philox::gen(a.ctrl->seed ^ 0x51ed270b1ULL, (uint32_t)r, (uint32_t)(g0 + 1), (uint32_t)t.unit,
                          ((uint32_t)a.worker << 24) ^ (uint32_t)a.ctrl->step, rnd);
              q8[g0 + 1] = quant4_i8(a1, inv, rnd);
            }
            if (g0 == 0) sbase[slot2_scale_off(u.rows, rcap, n) + r] = rowmax;
          }
        }
        if (ef) {     // e += A - U diag(s) V^T on the row's n elements
          float* er = residual + u.w_off + r * u.rs;
          for (int c = 0; c < n; ++c)
            er[(long long)c * u.cs] += __bfloat162float(row[(long long)c * u.cs]) -
                                       ef_recon(ust + tid, sv + c * V2_RCAP_MAX, count);
        }
      }
    }
  }

  // ---- completion: the last CTA publishes flag[group][worker] = step on every owner -------------------
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    const unsigned int old = atomicAdd(a.group_counter, 1u);
    if (old == gridDim.x - 1) {
      *a.group_counter = 0;
      __threadfence_system();
      const int step = a.ctrl->step;
      for (int o = 0; o < a.n_owners; ++o)
        st_release_sys(a.sig_peer[o] + SIG_PUSH + a.group * MAX_WORKERS + a.worker, step);
      if (a.tstats != nullptr) {
        const long long now = globaltimer_ns();
        if (a.timed) a.tstats[5] += now - a.tstats[9 + a.group];      // encode + project of this group
        if (a.final_group) a.tstats[8] += now - a.tstats[6];          // step start -> last push published
      }
    }
  }
}

__global__ void __launch_bounds__(ENC_THREADS) v2_project_kernel(const ProjArgs a) { project<false>(a, nullptr, 0); }
// error feedback: the same encode plus the residual epilogue
__global__ void __launch_bounds__(ENC_THREADS, 2) v2_project_ef_kernel(const ProjArgs a, float* residual,
                                                                        int ef_owner) {
  project<true>(a, residual, ef_owner);
}

// flag-only push of a group that has no encode tiles (dense-only configurations)
__global__ void v2_signal_kernel(int* const* sig_peer, int n_owners, int group, int worker, const Ctrl2* ctrl) {
  if (threadIdx.x == 0) {
    __threadfence_system();
    const int step = ctrl->step;
    for (int o = 0; o < n_owners; ++o) st_release_sys(sig_peer[o] + SIG_PUSH + group * MAX_WORKERS + worker, step);
  }
}

extern "C" {

int atomo_v2_unit_bytes() { return (int)sizeof(Unit2); }
int atomo_v2_ctrl_bytes() { return (int)sizeof(Ctrl2); }
int atomo_v2_enc_smem() { return ENC_SMEM; }

void atomo_v2_launch_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                            float* gpart, unsigned int* unit_counters, float* vsel, int* selcount, float* sigma_out,
                            float* const* arena_peer, int n_owners, long long arena_floats, void* stage,
                            const void* ctrl, const float* ext_uniforms, float* vprev, int max_sweeps,
                            int random_sample, int waterfill, int systematic, int worker, int resample_empty,
                            int flags, long long* tstats, int group, cudaStream_t stream) {
  if (ntiles <= 0) return;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(v2_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM);
    cudaFuncSetAttribute(v2_project_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PROJ_SMEM);
    cudaFuncSetAttribute(v2_project_ef_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PROJ_EF_SMEM);
    attr = true;
  }
  EncArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr; a.gpart = gpart;
  a.unit_counters = unit_counters; a.vsel = vsel; a.selcount = selcount; a.sigma_out = sigma_out;
  a.arena_peer = arena_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.stage = (__nv_bfloat16*)stage; a.ctrl = (const Ctrl2*)ctrl; a.ext_uniforms = ext_uniforms;
  a.vprev = vprev; a.max_sweeps = max_sweeps; a.flags = flags; a.tstats = tstats; a.group = group;
  a.cfg = EncCfg{random_sample, waterfill, systematic, worker, resample_empty};
  v2_encode_kernel<<<ntiles, ENC_THREADS, ENC_SMEM, stream>>>(a);
}

void atomo_v2_launch_project(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                             const float* vsel, const int* selcount, float* const* arena_peer, int* const* sig_peer,
                             int n_owners, long long arena_floats, int worker, int group, void* ctrl,
                             unsigned int* group_counter, int flags, long long* tstats, int final_group, int timed,
                             float* residual, int ef_owner, cudaStream_t stream) {
  if (ntiles <= 0) {
    v2_signal_kernel<<<1, 32, 0, stream>>>(sig_peer, n_owners, group, worker, (const Ctrl2*)ctrl);
    return;
  }
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(v2_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM);
    cudaFuncSetAttribute(v2_project_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PROJ_SMEM);
    cudaFuncSetAttribute(v2_project_ef_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PROJ_EF_SMEM);
    attr = true;
  }
  ProjArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr; a.vsel = vsel;
  a.selcount = selcount; a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners;
  a.arena_floats = arena_floats; a.worker = worker; a.group = group; a.ctrl = (Ctrl2*)ctrl;
  a.group_counter = group_counter; a.flags = flags; a.tstats = tstats; a.final_group = final_group; a.timed = timed;
  if (residual != nullptr) v2_project_ef_kernel<<<ntiles, ENC_THREADS, PROJ_EF_SMEM, stream>>>(a, residual, ef_owner);
  else v2_project_kernel<<<ntiles, ENC_THREADS, PROJ_SMEM, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
