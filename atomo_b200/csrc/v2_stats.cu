// Estimator statistics of the bf16 engine (sm_90a): per coded unit and step, the squared norm of the bf16 gradient,
// the expected squared error of the code given that gradient, the expected and the realized atom counts and, for
// TernGrad, the clip bias.  One launch per backward group, on the encode stream after the group's push, so the
// gradient, this step's sigma / selcount / L1 / clip and the worker's slot headers and norms are all live.
//
// The atoms of every code here are orthogonal and sampled independently (or, for systematic sampling, with the same
// marginals), so the error given the gradient has a closed form and the statistics are exact, not sampled:
//   spectral (SLAB / MAT):  sum over atoms of sigma_i^2 (1/p_i - 1), p_i of spectral_probs(); top-k: the dropped
//                           sigma_i^2.  sigma is the engine's (sorted) spectrum of this step.
//   entry-wise:             sum g_i^2 (1/p_i - 1), p_i = min(1, |g_i| * k) with the encoder's fp32 k = s / L1.
//   QSGD / TernGrad:        sum (nrm/s)^2 f_i (1 - f_i) per bucket, f_i the fractional part of s |v_i| / nrm, with
//                           the encoder's fp32 bucket norm (read back from the slot), in fp64; TernGrad on the
//                           clipped values v_i, plus the clip bias sum (v_i - g_i)^2 as a separate number.
//
//   v2_code_stats_kernel  one CTA per encode tile: fp64 partials of the tile (fixed warp / lane order); the last
//                         tile of each unit (unit counter) adds them in tile order, adds the spectral terms, and
//                         accumulates into acc[unit], so the sums have the same bits on every run.
#include "spectral_sample.cuh"
#include "v2_common.cuh"

namespace atomo {
namespace v2 {

constexpr int ST_THREADS = 256;
constexpr int ST_WARPS = ST_THREADS / 32;
constexpr int ST_PART = 5;              // per tile: gsq, mse, exp_atoms, bias_sq, realized atoms
constexpr int ST_ACC = 7;               // per unit: the five sums, realized atoms rounded up to U's groups of 4, steps
constexpr int ST_MAX_BUCKETS = 4096 / 32;

struct StatArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  int tile0;                   // global index of tiles[0] (partials are indexed by global encode tile)
  const long long* gptr;       // gradient base pointers (bf16), one per weight tensor
  const float* sigma;          // spectral: [n_coded][64] sorted singular values of this step
  const int* selcount;         // spectral: atoms selected per unit
  const double* l1;            // entry-wise: L1 norm per unit
  const float* clip;           // TernGrad: clip per unit
  float* const* arena_peer;    // [n_owners] arena base inside each owner (entry headers, QSGD norms)
  int n_owners;
  long long arena_floats;
  int worker;
  int random_sample, waterfill;
  double* partials;            // [n_enc_tiles][ST_PART]
  unsigned int* unit_counters; // [n_coded]
  double* acc;                 // [n_coded][ST_ACC]
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(ST_THREADS) v2_code_stats_kernel(const StatArgs a) {
  __shared__ double red[4][ST_WARPS];
  __shared__ float s_norm[ST_MAX_BUCKETS];
  __shared__ float s_prob[V2_MAX_COLS];
  __shared__ int s_order[V2_MAX_COLS];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  if (u.kind != KIND_SLAB && u.kind != KIND_MAT && u.kind != KIND_ENTRY && u.kind != KIND_QSGD) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
  const int jt = t.owner;      // encode tiles: index of the tile inside its unit (= PS tile for QSGD / entry units)
  const float* slot = a.arena_peer[(u.own0 + jt) % a.n_owners] + (long long)a.worker * a.arena_floats + u.slot_off;
  double gsq = 0.0, mse = 0.0, ex = 0.0, bias = 0.0, real = 0.0;

  if (u.kind == KIND_SLAB) {
    const long long n = (long long)t.b * u.K * u.I;
    const __nv_bfloat16* src = gb + (long long)t.a * u.K * u.I;
    for (long long i = tid; i < n; i += ST_THREADS) {
      const double x = (double)__bfloat162float(src[i]);
      gsq = fma(x, x, gsq);
    }
  } else if (u.kind == KIND_MAT) {
    const int n = t.b * u.cols;
    for (int e = tid; e < n; e += ST_THREADS) {
      const int r = e / u.cols, c = e - r * u.cols;
      const double x = (double)__bfloat162float(gb[(long long)(t.a + r) * u.rs + (long long)c * u.cs]);
      gsq = fma(x, x, gsq);
    }
  } else if (u.kind == KIND_ENTRY) {
    // the encoder's k = s / L1 (v2_entry_encode_kernel); L1 == 0 (or NaN) keeps nothing
    const double L1 = a.l1[u.ts_index];
    const float k = L1 > 0.0 ? (float)((double)u.budget / L1) : 0.f;
    const __nv_bfloat16* src = gb + t.a;
    for (int i = tid; i < t.b; i += ST_THREADS) {
      const float x = __bfloat162float(src[i]);
      const double xd = (double)x, x2 = xd * xd;
      gsq += x2;
      const float p = fabsf(x) * k;
      if (p >= 1.f) {
        ex += 1.0;
      } else if (p > 0.f) {
        ex += (double)p;
        mse += x2 * (1.0 / (double)p - 1.0);
      } else {
        mse += x2;
      }
    }
    if (tid == 0) real = (double)ld_cg_i(reinterpret_cast<const int*>(slot + entry_hdr_off(jt)) + 1);
  } else {
    // QSGD / TernGrad: every element travels; the error is the stochastic rounding's
    const int bucket = u.K, levels = (1 << u.I) - 1;
    const bool tern = u.rs != 0;
    const float clip = tern ? a.clip[u.ts_index] : 0.f;
    const int kb0 = t.a / bucket, nbt = (t.b + bucket - 1) / bucket;
    for (int kb = tid; kb < nbt; kb += ST_THREADS) s_norm[kb] = ld_cg_f(slot + qsgd_norms_off(u.n_ps) + kb0 + kb);
    __syncthreads();
    const __nv_bfloat16* src = gb + t.a;
    for (int i = tid; i < t.b; i += ST_THREADS) {
      const float x = __bfloat162float(src[i]);
      const float v = (tern && clip > 0.f) ? fminf(fmaxf(x, -clip), clip) : x;
      const double xd = (double)x, vd = (double)v;
      gsq = fma(xd, xd, gsq);
      bias = fma(vd - xd, vd - xd, bias);
      const double nrm = (double)s_norm[i / bucket];
      if (nrm > 0.0) {
        const double av = fmin(fabs(vd) * levels / nrm, (double)levels);
        const double f = av - floor(av), sc = nrm / levels;
        mse += sc * sc * f * (1.0 - f);
      }
    }
    if (tid == 0) ex = real = (double)t.b;
  }

  // ---- tile sums in a fixed order, then the unit's last tile combines the tiles in tile order ----------------
  gsq = warp_sum_d(gsq); mse = warp_sum_d(mse); ex = warp_sum_d(ex); bias = warp_sum_d(bias);
  if (lane == 0) { red[0][warp] = gsq; red[1][warp] = mse; red[2][warp] = ex; red[3][warp] = bias; }
  __syncthreads();
  if (tid == 0) {
    double* p = a.partials + (long long)ST_PART * (a.tile0 + blockIdx.x);
    for (int f = 0; f < 4; ++f) {
      double s = 0.0;
      for (int w = 0; w < ST_WARPS; ++w) s += red[f][w];
      p[f] = s;
    }
    p[4] = real;
    __threadfence();
    const unsigned int old = atomicAdd(&a.unit_counters[u.ts_index], 1u);
    s_last = (old == (unsigned int)u.n_enc - 1u) ? 1 : 0;
    if (s_last) a.unit_counters[u.ts_index] = 0;
  }
  __syncthreads();
  if (!s_last || tid != 0) return;
  __threadfence();
  double sum[ST_PART] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < u.n_enc; ++k) {
    const double* pk = a.partials + (long long)ST_PART * (u.enc_tile0 + k);
    for (int f = 0; f < ST_PART; ++f) sum[f] += __ldcg(pk + f);
  }
  double real4 = sum[4];
  if (u.kind == KIND_SLAB || u.kind == KIND_MAT) {
    // the sampler's probabilities on the sorted spectrum (order = identity); U is stored in groups of 4 atoms
    const int n = u.cols;
    const float* sg = a.sigma + (long long)u.ts_index * V2_MAX_COLS;
    float total = 0.f;
    for (int i = 0; i < n; ++i) total += sg[i];
    const float smax = sg[0];
    double m = 0.0, e = 0.0;
    if (!(smax >= 1e-6f)) {
      e = 1.0;                                       // degenerate spectrum: atom 0 with probability 1
      for (int i = 1; i < n; ++i) m += (double)sg[i] * sg[i];
    } else if (!a.random_sample) {
      const int k = min(min(u.budget > 0.f ? (int)u.budget : n, n), u.rcap);
      e = k;
      for (int i = k; i < n; ++i) m += (double)sg[i] * sg[i];
    } else {
      for (int i = 0; i < n; ++i) s_order[i] = i;
      spectral_probs(sg, s_order, n, u.budget, a.waterfill, total, smax, s_prob);
      for (int i = 0; i < n; ++i) {
        const double p = (double)s_prob[i], s2 = (double)sg[i] * sg[i];
        e += p;
        m += p > 0.0 ? s2 * (1.0 / p - 1.0) : s2;
      }
    }
    const int cnt = a.selcount[u.ts_index];
    sum[1] = m; sum[2] = e; sum[4] = (double)cnt;
    real4 = (double)min(u.rcap, (cnt + 3) & ~3);
  }
  double* acc = a.acc + (long long)ST_ACC * u.ts_index;
  for (int f = 0; f < ST_PART; ++f) acc[f] += sum[f];
  acc[5] += real4;
  acc[6] += 1.0;
}

extern "C" {

int atomo_v2_stats_fields() { return ST_ACC; }
int atomo_v2_stats_partials() { return ST_PART; }

void atomo_v2_launch_code_stats(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                const float* sigma, const int* selcount, const double* l1, const float* clip,
                                float* const* arena_peer, int n_owners, long long arena_floats, int worker,
                                int random_sample, int waterfill, double* partials, unsigned int* unit_counters,
                                double* acc, cudaStream_t stream) {
  if (ntiles <= 0) return;
  StatArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr;
  a.sigma = sigma; a.selcount = selcount; a.l1 = l1; a.clip = clip; a.arena_peer = arena_peer;
  a.n_owners = n_owners; a.arena_floats = arena_floats; a.worker = worker; a.random_sample = random_sample;
  a.waterfill = waterfill; a.partials = partials; a.unit_counters = unit_counters; a.acc = acc;
  v2_code_stats_kernel<<<ntiles, ST_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
