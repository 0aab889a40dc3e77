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
//                      publishes flag[group][worker] = step on every owner with st.release.sys.
#include "v2_common.cuh"

namespace atomo {
namespace v2 {

constexpr int ENC_THREADS = 256;
constexpr int ENC_HDR = 128;
constexpr int ENC_TILE_BYTES = 36 * 1024;       // tile buffer; reused for G / V (2 x 64 x 65 floats) in the eig phase
constexpr int ENC_RED_BYTES = 64 * 64 * 4;
constexpr int ENC_SMEM = ENC_HDR + ENC_TILE_BYTES + ENC_RED_BYTES;
constexpr int GS2 = V2_MAX_COLS + 1;
constexpr int MAX_SWEEPS2 = 12;

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

__device__ __forceinline__ void rr_pair2(int ne, int rnd, int k, int& p, int& q) {
  const int m = ne - 1;
  int a, b;
  if (k == 0) { a = rnd % m; b = m; }
  else { a = (rnd + k) % m; b = (rnd - k + m) % m; }
  p = min(a, b); q = max(a, b);
}

// ------------------------------------------------------------------------------------------------------
// Eigen-decomposition of the unit's Gram + atom sampling (svd.py:49-67 semantics, see csrc/svd_kernels.cu for
// the round-1 stand-alone version).  Runs in the LAST encode CTA of the unit; G / V live in the tile buffer.
// ------------------------------------------------------------------------------------------------------
__device__ void eig_sample_unit(const EncArgs& a, const Unit2& u, int unit_id, float* G, float* V, float* Tbuf) {
  __shared__ float rc[V2_MAX_COLS / 2], rs[V2_MAX_COLS / 2];
  __shared__ int rp[V2_MAX_COLS / 2], rq[V2_MAX_COLS / 2];
  __shared__ float sig[V2_MAX_COLS], prob[V2_MAX_COLS], uni[V2_MAX_COLS];
  __shared__ int order[V2_MAX_COLS];
  __shared__ int sel[V2_RCAP_MAX];
  __shared__ float selscale[V2_RCAP_MAX];
  __shared__ int s_maxrel;
  __shared__ float s_gmax;
  __shared__ int s_count, s_done;

  const int n = u.cols, tid = threadIdx.x, nthr = blockDim.x;
  const int step = a.ctrl->step;
  const int ts = u.ts_index;
  const int ne = n + (n & 1), npairs = ne >> 1;
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
    G[i * GS2 + j] = s;
    float v0 = (i == j) ? 1.f : 0.f;
    if (warm && i < n && j < n) v0 = vp[i * n + j];
    V[i * GS2 + j] = v0;
  }
  if (warm) {
    float* T = Tbuf;   // n x n scratch (the Gram reduction buffer of the tile phase)
    __syncthreads();
    for (int e = tid; e < n * n; e += nthr) {       // T = G V0
      const int i = e / n, j = e - i * n;
      float acc = 0.f;
      for (int k = 0; k < n; ++k) acc = fmaf(G[i * GS2 + k], V[k * GS2 + j], acc);
      T[e] = acc;
    }
    __syncthreads();
    for (int e = tid; e < n * n; e += nthr) {       // G0 = V0^T T, symmetrized
      const int i = e / n, j = e - i * n;
      if (i <= j) {
        float x = 0.f, y = 0.f;
        for (int k = 0; k < n; ++k) {
          x = fmaf(V[k * GS2 + i], T[k * n + j], x);
          y = fmaf(V[k * GS2 + j], T[k * n + i], y);
        }
        const float v = 0.5f * (x + y);
        G[i * GS2 + j] = v;
        G[j * GS2 + i] = v;
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    float g = 0.f;
    for (int i = 0; i < n; ++i) g = fmaxf(g, fabsf(G[i * GS2 + i]));
    s_gmax = g;
  }
  __syncthreads();
  const float gmax = s_gmax;
  if (n > 1 && gmax > 0.f) {
    // warm: a.max_sweeps refinement sweeps track the slowly drifting basis; cold (first step / periodic reset): full solve
    const int sweeps = (warm && a.max_sweeps > 0) ? min(a.max_sweeps, MAX_SWEEPS2) : MAX_SWEEPS2;
    for (int sweep = 0; sweep < sweeps; ++sweep) {
      if (tid == 0) s_maxrel = 0;
      __syncthreads();
      for (int rnd = 0; rnd < ne - 1; ++rnd) {
        if (tid < npairs) {
          int p, q;
          rr_pair2(ne, rnd, tid, p, q);
          float c = 1.f, s = 0.f;
          const float apq = G[p * GS2 + q], app = G[p * GS2 + p], aqq = G[q * GS2 + q];
          const float scale = sqrtf(fabsf(app * aqq));
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
        // two-sided update of the 2x2 blocks G[{p1,q1}][{p2,q2}] ...
        {
          int k1 = tid / npairs, k2 = tid - k1 * npairs;
          const int dk1 = nthr / npairs, dk2 = nthr - dk1 * npairs;
          while (k1 < npairs) {
            const int p1 = rp[k1], q1 = rq[k1], p2 = rp[k2], q2 = rq[k2];
            const float c1 = rc[k1], s1 = rs[k1], c2 = rc[k2], s2 = rs[k2];
            const float x = G[p1 * GS2 + p2], y = G[p1 * GS2 + q2], z = G[q1 * GS2 + p2], w = G[q1 * GS2 + q2];
            const float ra = c1 * x - s1 * z, rb = c1 * y - s1 * w;
            const float rc_ = s1 * x + c1 * z, rd = s1 * y + c1 * w;
            G[p1 * GS2 + p2] = c2 * ra - s2 * rb;
            G[p1 * GS2 + q2] = s2 * ra + c2 * rb;
            G[q1 * GS2 + p2] = c2 * rc_ - s2 * rd;
            G[q1 * GS2 + q2] = s2 * rc_ + c2 * rd;
            k1 += dk1; k2 += dk2;
            if (k2 >= npairs) { k2 -= npairs; ++k1; }
          }
        }
        // ... and the column rotations of V (row i, pair k)
        {
          int k = tid / ne, i = tid - k * ne;
          const int dk = nthr / ne, di = nthr - dk * ne;
          while (k < npairs) {
            const int p = rp[k], q = rq[k];
            const float c = rc[k], sn = rs[k];
            const float vp_ = V[i * GS2 + p], vq = V[i * GS2 + q];
            V[i * GS2 + p] = c * vp_ - sn * vq;
            V[i * GS2 + q] = sn * vp_ + c * vq;
            k += dk; i += di;
            if (i >= ne) { i -= ne; ++k; }
          }
        }
        __syncthreads();
      }
      // Every thread must have read s_maxrel before thread 0 resets it for the next sweep: without this barrier a
      // slow warp can see the reset value, leave the loop alone and desynchronise every barrier that follows
      // (observed as random illegal-address / illegal-instruction faults once this kernel shared SMs with cuDNN).
      const float mr = __int_as_float(s_maxrel);
      __syncthreads();
      if (mr < 1e-3f) break;
    }
  }
  __syncthreads();
  if (tid < n) {
    float d = G[tid * GS2 + tid];
    if (!(d >= 0.f) || !(d <= 3.0e38f)) {          // NaN / Inf / negative: flag it, treat the direction as empty
      if (!(d > -1e-3f * gmax)) atomicOr(const_cast<int*>(&a.ctrl->error), ERR2_NONFINITE);
      d = 0.f;
    }
    sig[tid] = sqrtf(d);
    order[tid] = tid;
  }
  __syncthreads();
  if (tid < n) {
    const float me = sig[tid];
    int rk = 0;
    for (int j = 0; j < n; ++j) {
      const float o = sig[j];
      rk += (o > me) || (o == me && j < tid);
    }
    order[rk] = tid;
  }
  __syncthreads();

  const int rcap = u.rcap;
  const float budget = u.budget;
  if (tid == 0) {
    float total = 0.f;
    for (int i = 0; i < n; ++i) total += sig[i];
    const float smax = sig[order[0]];
    int count = 0;
    if (!(smax >= 1e-6f)) {
      sel[0] = order[0]; selscale[0] = 1.f; count = 1;
      for (int i = 0; i < n; ++i) prob[i] = 0.f;
      prob[order[0]] = 1.f;
      s_done = 1;
    } else if (!a.cfg.random_sample) {
      const int k = min(min(budget > 0.f ? (int)budget : n, n), rcap);
      for (int x = 0; x < k; ++x) { sel[x] = order[x]; selscale[x] = 1.f; }
      count = k;
      s_done = 1;
    } else {
      if (budget <= 0.f) {
        for (int i = 0; i < n; ++i) prob[i] = fminf(sig[i] / smax, 1.f);
      } else if (!a.cfg.waterfill) {
        for (int i = 0; i < n; ++i) prob[i] = fminf(budget * sig[i] / total, 1.f);
      } else {
        const float bud = fminf(budget, (float)n);
        float rest = total;
        int pinned = 0;
        while (pinned < n) {
          const float s0 = sig[order[pinned]];
          if (rest > 0.f && (bud - pinned) * s0 >= rest && (bud - pinned) > 0.f) { rest -= s0; ++pinned; }
          else break;
        }
        for (int k = 0; k < n; ++k) {
          const int i = order[k];
          prob[i] = (k < pinned) ? 1.f : (rest > 0.f ? fminf((bud - pinned) * sig[i] / rest, 1.f) : 0.f);
        }
      }
      s_done = 0;
    }
    s_count = count;
  }
  __syncthreads();
  if (!s_done) {
    for (int attempt = 0; attempt < 16 && !s_done; ++attempt) {
      if (tid < n) {
        float x;
        if (a.ext_uniforms != nullptr && attempt == 0) {
          x = a.ext_uniforms[(long long)ts * V2_MAX_COLS + tid];
        } else {
          uint32_t r4[4];
          Philox::gen(a.ctrl->seed, (uint32_t)tid, (uint32_t)attempt, (uint32_t)unit_id,
                      ((uint32_t)a.cfg.worker << 24) ^ (uint32_t)step, r4);
          x = Philox::to_uniform(r4[0]);
        }
        uni[tid] = x;
      }
      __syncthreads();
      if (tid == 0) {
        int count = 0;
        bool overflow = false;
        if (a.cfg.systematic) {
          const float x = uni[0];
          float c = 0.f;
          for (int k = 0; k < n; ++k) {
            const int i = order[k];
            const float lo = floorf(c + x);
            c += prob[i];
            const float hi = floorf(c + x);
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
        if ((count > 0 || !a.cfg.resample_empty) && !overflow) { s_count = count; s_done = 1; }
      }
      __syncthreads();
    }
    if (!s_done) {
      if (tid == 0) {
        const int k = min(max((int)budget, 1), min(n, rcap));
        for (int x = 0; x < k; ++x) { sel[x] = order[x]; selscale[x] = 1.f / fmaxf(prob[order[x]], 1e-6f); }
        s_count = k; s_done = 1;
      }
      __syncthreads();
    }
  }
  const int count = s_count;

  // ---- publish: local projection basis, and header / s / V into every owner's slot (peer stores) ----
  float* vs = a.vsel + (long long)ts * V2_MAX_COLS * V2_RCAP_MAX;
  for (int e = tid; e < n * V2_RCAP_MAX; e += nthr) {
    const int c = e / V2_RCAP_MAX, x = e - c * V2_RCAP_MAX;
    float v = 0.f;
    if (x < count) {
      const int i = sel[x];
      v = (sig[i] > 1e-7f * sig[order[0]]) ? V[c * GS2 + i] / sig[i] : 0.f;
    }
    vs[e] = v;
  }
  if (tid == 0) a.selcount[ts] = count;
  if (vp != nullptr)
    for (int e = tid; e < n * n; e += nthr) vp[e] = V[(e / n) * GS2 + (e % n)];
  if (a.sigma_out != nullptr && tid < n) a.sigma_out[(long long)ts * V2_MAX_COLS + tid] = sig[order[tid]];
  // header / s / V go to every owner's slot.  Only warp 0 stores (and fences): a system-scope fence per thread
  // of the CTA costs microseconds, one per lane of a single warp is one instruction.
  if (tid < 32) {
    for (int o = 0; o < a.n_owners; ++o) {
      float* slot = a.arena_peer[o] + (long long)a.cfg.worker * a.arena_floats + u.slot_off;
      for (int x = tid; x < rcap; x += 32) slot[4 + x] = (x < count) ? sig[sel[x]] * selscale[x] : 0.f;
      float* vout = slot + 4 + rcap;
      for (int e = tid; e < rcap * n; e += 32) {
        const int x = e / n, c = e - x * n;
        vout[e] = (x < count) ? V[c * GS2 + sel[x]] : 0.f;
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
    float* V = G + V2_MAX_COLS * GS2;
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

__global__ void __launch_bounds__(ENC_THREADS) v2_project_kernel(const ProjArgs a) {
  uint64_t* mbar = reinterpret_cast<uint64_t*>(enc_smem);
  uint32_t* tile = reinterpret_cast<uint32_t*>(enc_smem + ENC_HDR);
  float* vs = reinterpret_cast<float*>(enc_smem + ENC_HDR + ENC_TILE_BYTES);
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x;

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
                             cudaStream_t stream) {
  if (ntiles <= 0) {
    v2_signal_kernel<<<1, 32, 0, stream>>>(sig_peer, n_owners, group, worker, (const Ctrl2*)ctrl);
    return;
  }
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(v2_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ENC_SMEM);
    cudaFuncSetAttribute(v2_project_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PROJ_SMEM);
    attr = true;
  }
  ProjArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr; a.vsel = vsel;
  a.selcount = selcount; a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners;
  a.arena_floats = arena_floats; a.worker = worker; a.group = group; a.ctrl = (Ctrl2*)ctrl;
  a.group_counter = group_counter; a.flags = flags; a.tstats = tstats; a.final_group = final_group; a.timed = timed;
  v2_project_kernel<<<ntiles, ENC_THREADS, PROJ_SMEM, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
