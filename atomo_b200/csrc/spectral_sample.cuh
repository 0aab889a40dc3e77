// Eigen-decomposition of a unit's Gram matrix and ATOMO atom sampling (svd.py:49-67 semantics): the core shared by
// the fp32 engine's eig_sample_kernel (svd_kernels.cu) and the bf16 engine's v2_encode_kernel (v2_encode.cu).
#pragma once
#include "common.cuh"

namespace atomo {

constexpr int SPECTRAL_PITCH = TS_MAX_COLS + 1;  // padded row stride of G / V in shared memory
constexpr int JACOBI_MAX_SWEEPS = 12;

__device__ __forceinline__ void rr_pair(int ne, int rnd, int k, int& p, int& q) {
  // round-robin tournament over `ne` (even) players: ne/2 disjoint pairs per round
  const int m = ne - 1;
  int a, b;
  if (k == 0) { a = rnd % m; b = m; }
  else { a = (rnd + k) % m; b = (rnd - k + m) % m; }
  p = min(a, b); q = max(a, b);
}

// How a unit's atoms are drawn.
struct SampleCfg {
  float budget;               // expected number of atoms; <= 0: p_i = sigma_i / sigma_max (svd.py:52)
  int rcap;                   // slot capacity in atoms (<= RCAP_MAX)
  int random_sample;          // 0: keep the top-min(budget, n, rcap) atoms (svd.py:109-113)
  int waterfill;              // 0: the reference's clip p_i = min(1, budget sigma_i / sum sigma); 1: water-filling
  int systematic;             // 0: independent Bernoulli; 1: systematic sampling
  int resample_empty;         // 1: redraw when nothing was selected (the reference's rule, svd.py:65-66)
  const float* ext_uniforms;  // tests: [row][TS_MAX_COLS] uniforms for the first draw instead of Philox, or nullptr
  const unsigned long long* seed;  // Philox key, read at each draw; counter = (thread, draw, unit_id, tag)
  int unit_id;
  uint32_t tag;
};

// Inclusion probabilities of a randomly sampled unit (svd.py:49-67), written by one thread: prob[i] for the n singular
// values sig[i], where order[k] is the index of the k-th largest, total their sum and smax the largest (>= 1e-6).
// budget <= 0: p_i = sigma_i / sigma_max; else the reference's clip p_i = min(1, budget sigma_i / total), or
// water-filling, which pins the largest atoms to 1.  Shared by the sampler below and the estimator statistics
// (v2_stats.cu), so both see the same p_i.
__device__ __forceinline__ void spectral_probs(const float* sig, const int* order, int n, float budget, int waterfill,
                                               float total, float smax, float* prob) {
  if (budget <= 0.f) {
    for (int i = 0; i < n; ++i) prob[i] = fminf(sig[i] / smax, 1.f);
  } else if (!waterfill) {
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
}

// The core's results, in shared memory; valid until the caller's kernel ends.
struct Spectrum {
  int count;              // atoms selected
  const float* sig;       // sig[i] = sigma_i
  const int* order;       // order[k] = index of the k-th largest sigma
  const int* sel;         // sel[a] = index of atom a
  const float* selscale;  // selscale[a] = 1 / p of atom a
};

// One CTA per unit.  On entry, after a barrier, G holds the n x n Gram matrix, padded to an even size with a zero row
// and column, and V the starting basis, both with row pitch SPECTRAL_PITCH: the identity, or (`warm`) a previous basis
// with G already rotated into it, which then gets at most `max_sweeps` sweeps if that is > 0.  Jacobi leaves the
// eigenvalues on G's diagonal and the eigenvectors in V's columns; then the atoms are sampled and the projection basis
// of the second pass is stored in the unit's `row` of vsel:
//   vsel[row][c*RCAP_MAX + a] = V[c][sel_a] / sigma_a   (so U = A vsel), zero for a >= count.
// flag_nonfinite: a NaN / Inf / negative eigenvalue becomes an empty direction, and one that is not just rounding
// below zero raises `err_bit` in `*err`.  Otherwise sigma = sqrt(max(lambda, 0)).  Callers pass a constant, which the
// inlining folds.  (A template parameter would move this function's __shared__ arrays behind the calling kernel's
// own in the shared-memory layout, and with them every address in the kernel.)
__device__ __forceinline__ Spectrum eig_sample(float* G, float* V, int n, bool warm, int max_sweeps,
                                               const SampleCfg& cfg, int row, float* vsel, int* err, int err_bit,
                                               bool flag_nonfinite) {
  __shared__ float rc[TS_MAX_COLS / 2], rs[TS_MAX_COLS / 2];
  __shared__ int rp[TS_MAX_COLS / 2], rq[TS_MAX_COLS / 2];
  __shared__ float sig[TS_MAX_COLS], prob[TS_MAX_COLS], uni[TS_MAX_COLS];
  __shared__ int order[TS_MAX_COLS];
  __shared__ int sel[RCAP_MAX];
  __shared__ float selscale[RCAP_MAX];
  __shared__ int s_maxrel;
  __shared__ float s_gmax;
  __shared__ int s_count, s_done;

  const int tid = threadIdx.x, nthr = blockDim.x;
  const int ne = n + (n & 1), npairs = ne >> 1;

  // ---- cyclic Jacobi, round-robin (parallel) ordering, fused two-sided update ------------------
  // All ne/2 pairs of a round are disjoint, so G' = J^T G J decomposes into independent 2x2 blocks: block (k1,k2) =
  // J_k1^T * G[{p1,q1}][{p2,q2}] * J_k2, each computed by one thread, with one barrier between "compute rotations" and
  // "apply" and none between the row and column halves.  The padded dummy index only ever meets zeros, so its
  // rotations are the identity.
  if (tid == 0) {
    float g = 0.f;
    for (int i = 0; i < n; ++i) g = fmaxf(g, fabsf(G[i * SPECTRAL_PITCH + i]));
    s_gmax = g;
  }
  __syncthreads();
  const float gmax = s_gmax;
  if (n > 1 && gmax > 0.f) {
    const int sweeps = (warm && max_sweeps > 0) ? min(max_sweeps, JACOBI_MAX_SWEEPS) : JACOBI_MAX_SWEEPS;
    for (int sweep = 0; sweep < sweeps; ++sweep) {
      if (tid == 0) s_maxrel = 0;
      __syncthreads();
      for (int rnd = 0; rnd < ne - 1; ++rnd) {
        if (tid < npairs) {
          int p, q;
          rr_pair(ne, rnd, tid, p, q);
          float c = 1.f, s = 0.f;
          const float apq = G[p * SPECTRAL_PITCH + q], app = G[p * SPECTRAL_PITCH + p], aqq = G[q * SPECTRAL_PITCH + q];
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
        // two-sided update of the 2x2 blocks G[{p1,q1}][{p2,q2}] ...
        {
          int k1 = tid / npairs, k2 = tid - k1 * npairs;
          const int dk1 = nthr / npairs, dk2 = nthr - dk1 * npairs;
          while (k1 < npairs) {
            const int p1 = rp[k1], q1 = rq[k1], p2 = rp[k2], q2 = rq[k2];
            const float c1 = rc[k1], s1 = rs[k1], c2 = rc[k2], s2 = rs[k2];
            const float x = G[p1 * SPECTRAL_PITCH + p2], y = G[p1 * SPECTRAL_PITCH + q2];
            const float z = G[q1 * SPECTRAL_PITCH + p2], w = G[q1 * SPECTRAL_PITCH + q2];
            // left: rows (p1,q1) <- J1^T
            const float ra = c1 * x - s1 * z, rb = c1 * y - s1 * w;
            const float rc_ = s1 * x + c1 * z, rd = s1 * y + c1 * w;
            // right: cols (p2,q2) <- J2
            G[p1 * SPECTRAL_PITCH + p2] = c2 * ra - s2 * rb;
            G[p1 * SPECTRAL_PITCH + q2] = s2 * ra + c2 * rb;
            G[q1 * SPECTRAL_PITCH + p2] = c2 * rc_ - s2 * rd;
            G[q1 * SPECTRAL_PITCH + q2] = s2 * rc_ + c2 * rd;
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
            const float vp_ = V[i * SPECTRAL_PITCH + p], vq = V[i * SPECTRAL_PITCH + q];
            V[i * SPECTRAL_PITCH + p] = c * vp_ - sn * vq;
            V[i * SPECTRAL_PITCH + q] = sn * vp_ + c * vq;
            k += dk; i += di;
            if (i >= ne) { i -= ne; ++k; }
          }
        }
        __syncthreads();
      }
      // Quadratic convergence: couplings below 1e-3 at the start of a sweep are ~1e-6 after it.  Every thread must
      // have read s_maxrel before thread 0 resets it for the next sweep: without this barrier a slow warp can see the
      // reset value, leave the loop alone and desynchronise every barrier that follows (observed as random
      // illegal-address / illegal-instruction faults once the encode shared SMs with cuDNN).
      const float mr = __int_as_float(s_maxrel);
      __syncthreads();
      if (mr < 1e-3f) break;
    }
  }
  __syncthreads();

  // ---- singular values, descending order (ties by index) ------------------------------------------
  if (tid < n) {
    float d = G[tid * SPECTRAL_PITCH + tid];
    if (flag_nonfinite) {
      if (!(d >= 0.f) || !(d <= 3.0e38f)) {
        if (!(d > -1e-3f * gmax)) atomicOr(err, err_bit);
        d = 0.f;
      }
    } else {
      d = fmaxf(d, 0.f);
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

  // ---- inclusion probabilities -------------------------------------------------------------------
  const int rcap = cfg.rcap;
  const float budget = cfg.budget;
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
      const int k = min(min(budget > 0.f ? (int)budget : n, n), rcap);
      for (int x = 0; x < k; ++x) { sel[x] = order[x]; selscale[x] = 1.f; }
      count = k;
      s_done = 1;
    } else {
      spectral_probs(sig, order, n, budget, cfg.waterfill, total, smax, prob);
      s_done = 0;
    }
    s_count = count;
  }
  __syncthreads();

  // ---- sampling: draws that overflow the slot (or are empty, with resample_empty) are redrawn -----------
  if (!s_done) {
    for (int attempt = 0; attempt < 16 && !s_done; ++attempt) {
      if (tid < n) {
        float x;
        if (cfg.ext_uniforms != nullptr && attempt == 0) {
          x = cfg.ext_uniforms[(long long)row * TS_MAX_COLS + tid];
        } else {
          uint32_t r4[4];
          Philox::gen(*cfg.seed, (uint32_t)tid, (uint32_t)attempt, (uint32_t)cfg.unit_id, cfg.tag, r4);
          x = Philox::to_uniform(r4[0]);
        }
        uni[tid] = x;
      }
      __syncthreads();
      if (tid == 0) {
        int count = 0;
        bool overflow = false;
        if (cfg.systematic) {
          // one uniform, cumulative probabilities in descending-sigma order
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
        if ((count > 0 || !cfg.resample_empty) && !overflow) { s_count = count; s_done = 1; }
      }
      __syncthreads();
    }
    if (!s_done) {
      // pathological: deterministic fallback on the most probable atoms
      if (tid == 0) {
        const int k = min(max((int)budget, 1), min(n, rcap));
        for (int x = 0; x < k; ++x) { sel[x] = order[x]; selscale[x] = 1.f / fmaxf(prob[order[x]], 1e-6f); }
        s_count = k; s_done = 1;
      }
      __syncthreads();
    }
  }
  const int count = s_count;

  // ---- projection basis ------------------------------------------------------------------------------
  float* vs = vsel + (long long)row * TS_MAX_COLS * RCAP_MAX;
  for (int e = tid; e < n * RCAP_MAX; e += nthr) {
    const int c = e / RCAP_MAX, x = e - c * RCAP_MAX;
    float v = 0.f;
    if (x < count) {
      const int i = sel[x];
      // a (numerically) null direction has no left vector: emit a zero column instead of 1/0
      v = (sig[i] > 1e-7f * sig[order[0]]) ? V[c * SPECTRAL_PITCH + i] / sig[i] : 0.f;
    }
    vs[e] = v;
  }
  return Spectrum{count, sig, order, sel, selscale};
}

}  // namespace atomo
