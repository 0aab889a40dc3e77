// PowerSGD on the overlapped, sharded bf16 engine (sm_90a): one warm-started power step per weight matrix and step,
// pushed as a rank-r pair (P_hat, Q'), the owner-side reconstruction + optimizer step, and --code-stats.  The oracle is
// codings/powersgd.py; the geometry is ops/plan2.py (KIND_POWER).
//
// M is a weight gradient [O][C] in its physical (channels-last) order, read in place as bf16.  All factors are stored
// k-major (row k of P^T / P_hat^T has stride round4(O), of Q'^T / Q_w^T stride round4(C)) so a thread's 8 consecutive
// rows / columns of one factor column are two 16-byte loads.  Every sum runs in a fixed order: no float atomics.
//
//   v2_powersgd_encode_a_kernel  one CTA per PW_ENC_ROWS-row tile: P rows = M_tile Q_w (fp32, thread-private sums over
//                                8-column chunks, then a fixed butterfly + warp-order sum), P into the local scratch and
//                                an fp64 Gram partial per tile.  The unit's last tile (unit counter) sums the partials in
//                                tile order, factors G under the pivot rule and stores R^{-1}, the degenerate mask and
//                                the draw counter.  DENSE16 tiles get their staging copy here.
//   v2_powersgd_encode_b_kernel  one CTA per PW_COL_BLOCK-column block: P_hat = P R^{-1} (fp64 products, staged in shared
//                                memory), Q'[block] = M^T P_hat summed over all rows inside the CTA (warps take rows
//                                w, w + 8, ..., then a warp-order sum), so Q' has no cross-CTA partials.  Q' goes to the
//                                local scratch, to the unit's owner (every PS tile of a unit has the one owner own0, so
//                                Q' travels once) and, with re-drawn degenerate columns, to Q_w; block 0 stores P_hat.
//                                The unit's last block writes the PS tiles' step stamps; the last CTA of the launch
//                                publishes the push flag.
//   v2_powersgd_encode_ef_kernel error feedback (launched only with a residual): e += x - g_hat over pass-A tiles, g_hat
//                                with the owner's fmaf order.
//   v2_ps_powersgd_kernel        one launch per (group, owner): push wait / --num-aggregate mask / stale-slot check and
//                                fp32 vector tiles of v2_ps_common.cuh; per PW_PS_ROWS-row tile the counted workers'
//                                P_hat rows are staged in shared memory and sum_w sum_k P_hat_w[o][k] Q'_w[c][k] is
//                                accumulated with fmaf in worker order, then atom order, times 1/#counted, then the
//                                fused optimizer epilogue and the bf16 broadcast.  DENSE16 tiles: ps_dense16_tile.
//   v2_powersgd_code_stats_kernel --code-stats: per pass-A tile gsq = sum x^2 and mse = sum (x - g_hat)^2 in fp64 (the
//                                error of the code, exact); atoms = non-degenerate columns.  Tile-order sums.
//   v2_powersgd_init_kernel      Q_w = standard normals of draw 0 (engine construction, outside the graph).
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int PW_THREADS = 256;
constexpr int PW_WARPS = PW_THREADS / 32;
constexpr int PW_MAXR = 4;
constexpr int PW_ENC_ROWS = 8;
constexpr int PW_COL_BLOCK = 256;
constexpr int PW_PS_ROWS = 4;
constexpr int PW_GRAM = 16;
constexpr int PW_PH_CHUNK = 512;          // P_hat rows staged per round of pass B
constexpr double PW_PIVOT_RTOL = 1e-12;
constexpr unsigned long long PW_KEY_XOR = 0x70C5D1A3B2E49F17ULL;

// per PowerSGD unit (index ts_index), worker-local; all zero at construction
struct PwState {
  double rinv[16];      // R^{-1} [i][j], zero columns for degenerate j
  int mask;             // bit j: column j not degenerate
  int nonfinite;        // G had an Inf / NaN: zeros pushed, Q_w kept
  int draw;             // draw counter of the latest re-draw (0: the initial draw)
  unsigned int cnt_a;   // pass-A tiles done (self-resetting)
  unsigned int cnt_b;   // pass-B blocks done (self-resetting)
  int pad[3];
};
static_assert(sizeof(PwState) == 160, "PwState layout");

__host__ __device__ inline int pw_r4(int x) { return (x + 3) & ~3; }
// slot (floats, from Unit2::slot_off inside one worker arena): int32 stamp per PS tile | P_hat^T [r][round4(O)] |
// Q'^T [r][round4(C)]  (ops/plan2.py pw_phat_off / pw_q_off)
__host__ __device__ inline long long pw_phat_off(int n_ps) { return pw_r4(n_ps); }
__host__ __device__ inline long long pw_q_off(int n_ps, int rows, int r) {
  return pw_phat_off(n_ps) + (long long)r * pw_r4(rows);
}
// local scratch (from Unit2::gpart_off): P^T | P_hat^T [r][round4(O)] | Q'^T | Q_w^T [r][round4(C)]
struct PwScratch {
  float *p, *ph, *q, *qw;
  int op, cp;
};
__device__ __forceinline__ PwScratch pw_scratch(float* base, const Unit2& u) {
  PwScratch s;
  s.op = pw_r4(u.rows); s.cp = pw_r4(u.cols);
  s.p = base + u.gpart_off;
  s.ph = s.p + (long long)u.rcap * s.op;
  s.q = s.ph + (long long)u.rcap * s.op;
  s.qw = s.q + (long long)u.rcap * s.cp;
  return s;
}

// 8 bf16 of a row from column c (0 past n): one 16-byte load when the rows are 16-byte aligned and whole
__device__ __forceinline__ void pw_load8(const __nv_bfloat16* row, int c, int n, bool vec, float (&x)[8]) {
  if (vec && c + 8 <= n) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(row + c));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { x[2 * i] = bf16_lo(w[i]); x[2 * i + 1] = bf16_hi(w[i]); }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = (c + i < n) ? __bfloat162float(row[c + i]) : 0.f;
  }
}
// 8 floats from column c of a k-major factor row (16-byte aligned at c % 8 == 0), 0 past n
__device__ __forceinline__ void pw_loadf8(const float* p, int c, int n, float (&x)[8]) {
  if (c + 8 <= n) {
    const float4 a = *reinterpret_cast<const float4*>(p + c), b = *reinterpret_cast<const float4*>(p + c + 4);
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = (c + i < n) ? p[c + i] : 0.f;
  }
}

// standard normal k of column `col` for (seed, unit, draw): Box-Muller in fp64 (codings/powersgd.py normals)
__device__ __forceinline__ float pw_normal(unsigned long long seed, int unit, int col, int draw, int k) {
  uint32_t w[4];
  Philox::gen(seed ^ PW_KEY_XOR, (uint32_t)col, (uint32_t)unit, (uint32_t)draw, (uint32_t)(k >> 1), w);
  const uint32_t w0 = (k & 1) ? w[2] : w[0], w1 = (k & 1) ? w[3] : w[1];
  const double u1 = ((double)(w0 >> 8) + 1.0) / 16777216.0, u2 = (double)(w1 >> 8) / 16777216.0;
  return (float)(sqrt(-2.0 * log(u1)) * cos(2.0 * 3.141592653589793 * u2));
}

struct PwArgs {
  const Unit2* units;
  const Tile2* tiles;          // pass A / EF / stats: encode tiles; pass B: pw tiles (offset to the group's first)
  int ntiles;
  int tile0;                   // global index of tiles[0] (Gram / stats partials are indexed by global encode tile)
  const long long* gptr;
  float* scratch;              // the gpart region
  double* gram;                // [n_enc_tiles][PW_GRAM]
  PwState* state;              // [n_coded]
  __nv_bfloat16* stage;        // DENSE16 staging region of this worker
  float* const* arena_peer;
  int* const* sig_peer;
  int n_owners;
  long long arena_floats;
  int worker;
  int group;
  const Ctrl2* ctrl;
  unsigned int* group_counter;
  long long* tstats;
  int final_group;
  float* residual;
};

// ---- pass A: P = M Q_w, Gram partials, Cholesky of the unit's G ------------------------------------------------
__device__ void pw_factor(PwState* st, const double* gram, int n, int r) {
  double G[16];
  for (int i = 0; i < 16; ++i) G[i] = 0.0;
  for (int t = 0; t < n; ++t)                             // tile order: the same bits on every run
    for (int i = 0; i < 16; ++i) G[i] += __ldcg(gram + (long long)PW_GRAM * t + i);
  bool finite = true;
  double gmax = 0.0;
  for (int i = 0; i < r; ++i)
    for (int j = 0; j < r; ++j) finite = finite && isfinite(G[4 * i + j]);
  double L[16], R[16];
  for (int i = 0; i < 16; ++i) { L[i] = 0.0; R[i] = 0.0; }
  int mask = 0;
  if (finite) {
    for (int j = 0; j < r; ++j) gmax = fmax(gmax, G[5 * j]);
    const double tol = PW_PIVOT_RTOL * gmax;
    for (int j = 0; j < r; ++j) {
      double d = G[5 * j];
      for (int k = 0; k < j; ++k) d -= L[4 * j + k] * L[4 * j + k];
      if (!isfinite(d) || d <= tol || d == 0.0) continue;
      const double ljj = sqrt(d);
      L[5 * j] = ljj;
      for (int i = j + 1; i < r; ++i) {
        double s = G[4 * i + j];
        for (int k = 0; k < j; ++k) s -= L[4 * i + k] * L[4 * j + k];
        L[4 * i + j] = s / ljj;
      }
      for (int i = 0; i < r; ++i) {
        double s = (i == j) ? 1.0 : 0.0;
        for (int k = 0; k < j; ++k) s -= L[4 * j + k] * R[4 * i + k];
        R[4 * i + j] = s / ljj;
      }
      mask |= 1 << j;
    }
  }
  for (int i = 0; i < 16; ++i) st->rinv[i] = R[i];
  st->mask = mask;
  st->nonfinite = finite ? 0 : 1;
  if (finite && mask != (1 << r) - 1) st->draw += 1;      // degenerate columns are re-drawn in pass B
}

__global__ void __launch_bounds__(PW_THREADS) v2_powersgd_encode_a_kernel(const PwArgs a) {
  __shared__ float red[PW_WARPS][PW_ENC_ROWS * PW_MAXR];
  __shared__ float sp[PW_ENC_ROWS * PW_MAXR];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
  if (u.kind == KIND_DENSE16) {
    // staging copy of a dense bf16 gradient into the symmetric heap (the owners pull it from there)
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
  if (u.kind != KIND_POWER) return;
  const int r = u.rcap, C = u.cols, nr = t.b;
  const PwScratch s = pw_scratch(a.scratch, u);
  const __nv_bfloat16* row0 = gb + (long long)t.a * C;
  const bool vec = ((reinterpret_cast<uintptr_t>(gb) & 15) == 0) && (C & 7) == 0;
  float acc[PW_ENC_ROWS][PW_MAXR];
#pragma unroll
  for (int i = 0; i < PW_ENC_ROWS; ++i)
#pragma unroll
    for (int k = 0; k < PW_MAXR; ++k) acc[i][k] = 0.f;
  for (int c = 8 * tid; c < C; c += 8 * PW_THREADS) {
    float qv[PW_MAXR][8];
#pragma unroll
    for (int k = 0; k < PW_MAXR; ++k) {
      if (k < r) pw_loadf8(s.qw + (long long)k * s.cp, c, C, qv[k]);
      else
#pragma unroll
        for (int j = 0; j < 8; ++j) qv[k][j] = 0.f;
    }
#pragma unroll
    for (int i = 0; i < PW_ENC_ROWS; ++i) {
      if (i < nr) {
        float x[8];
        pw_load8(row0 + (long long)i * C, c, C, vec, x);
#pragma unroll
        for (int k = 0; k < PW_MAXR; ++k)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][k] = fmaf(x[j], qv[k][j], acc[i][k]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < PW_ENC_ROWS; ++i)
#pragma unroll
    for (int k = 0; k < PW_MAXR; ++k) {
      float v = acc[i][k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[warp][i * PW_MAXR + k] = v;
    }
  __syncthreads();
  if (tid < PW_ENC_ROWS * PW_MAXR) {
    float v = 0.f;
    for (int w = 0; w < PW_WARPS; ++w) v += red[w][tid];   // warp order
    const int i = tid / PW_MAXR, k = tid % PW_MAXR;
    if (i >= nr || k >= r) v = 0.f;
    sp[tid] = v;
    if (i < nr && k < r) s.p[(long long)k * s.op + t.a + i] = v;
  }
  __syncthreads();
  if (tid < PW_GRAM) {                                      // fp64 Gram partial, rows in order
    const int i = tid >> 2, j = tid & 3;
    double g = 0.0;
    for (int o = 0; o < nr; ++o) g += (double)sp[o * PW_MAXR + i] * (double)sp[o * PW_MAXR + j];
    a.gram[(long long)PW_GRAM * (a.tile0 + blockIdx.x) + tid] = g;
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    PwState* st = a.state + u.ts_index;
    const unsigned int old = atomicAdd(&st->cnt_a, 1u);
    s_last = (old == (unsigned int)u.n_enc - 1u) ? 1 : 0;
    if (s_last) {
      st->cnt_a = 0;
      __threadfence();
      pw_factor(st, a.gram + (long long)PW_GRAM * u.enc_tile0, u.n_enc, r);
    }
  }
}

// ---- pass B: P_hat, Q' = M^T P_hat, pushes, Q_w update, stamps, push flag ---------------------------------------
__device__ __forceinline__ float pw_phat(const PwScratch& s, const double* rinv, int r, int o, int j) {
  double v = 0.0;
  for (int i = 0; i < r; ++i) v += (double)s.p[(long long)i * s.op + o] * rinv[4 * i + j];
  return (float)v;
}

__global__ void __launch_bounds__(PW_THREADS, 1) v2_powersgd_encode_b_kernel(const PwArgs a) {
  __shared__ __align__(16) float sph[PW_MAXR][PW_PH_CHUNK];
  __shared__ float red[PW_WARPS][PW_MAXR][PW_COL_BLOCK];
  __shared__ double s_rinv[16];
  __shared__ int s_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int step = a.ctrl->step;
  if (a.ntiles > 0) {
    const Tile2 t = a.tiles[blockIdx.x];
    const Unit2 u = a.units[t.unit];
    const int r = u.rcap, C = u.cols, O = u.rows;
    const PwScratch s = pw_scratch(a.scratch, u);
    PwState* st = a.state + u.ts_index;
    const int mask = st->mask, nonfinite = st->nonfinite, draw = st->draw;
    if (tid < 16) s_rinv[tid] = nonfinite ? 0.0 : st->rinv[tid];
    const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
    const bool vec = ((reinterpret_cast<uintptr_t>(gb) & 15) == 0) && (C & 7) == 0;
    const int c = t.a + 8 * lane;                           // this lane's 8 columns
    float acc[PW_MAXR][8];
#pragma unroll
    for (int k = 0; k < PW_MAXR; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
    __syncthreads();
    for (int o0 = 0; !nonfinite && o0 < O; o0 += PW_PH_CHUNK) {
      const int n = min(PW_PH_CHUNK, O - o0);
      __syncthreads();                                      // the previous chunk is consumed
      for (int idx = tid; idx < n; idx += PW_THREADS)
#pragma unroll
        for (int k = 0; k < PW_MAXR; ++k) sph[k][idx] = k < r ? pw_phat(s, s_rinv, r, o0 + idx, k) : 0.f;
      __syncthreads();
      if (c < t.a + t.b) {
        for (int i = warp; i < n; i += PW_WARPS) {          // rows w, w + 8, ...: a fixed order per warp
          float x[8];
          pw_load8(gb + (long long)(o0 + i) * C, c, C, vec, x);
#pragma unroll
          for (int k = 0; k < PW_MAXR; ++k) {
            const float ph = sph[k][i];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[k][j] = fmaf(x[j], ph, acc[k][j]);
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < PW_MAXR; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) red[warp][k][8 * lane + j] = acc[k][j];
    __syncthreads();
    float* slot = a.arena_peer[u.own0] + (long long)a.worker * a.arena_floats + u.slot_off;   // the unit's owner
    const long long qoff = pw_q_off(u.n_ps, O, r);
    if (tid < t.b) {
      const int cc = t.a + tid;
      const unsigned long long seed = a.ctrl->seed;
      for (int k = 0; k < r; ++k) {
        float q = 0.f;
        for (int w = 0; w < PW_WARPS; ++w) q += red[w][k][tid];   // warp order
        if (nonfinite) q = 0.f;
        s.q[(long long)k * s.cp + cc] = q;
        if (!nonfinite) s.qw[(long long)k * s.cp + cc] = ((mask >> k) & 1) ? q : pw_normal(seed, t.unit, cc, draw, k);
        slot[qoff + (long long)k * s.cp + cc] = q;
      }
    }
    if (t.owner == 0) {                                     // block 0: P_hat, locally and to the unit's owner
      for (int o = tid; o < O; o += PW_THREADS) {
        for (int k = 0; k < r; ++k) {
          const float ph = nonfinite ? 0.f : pw_phat(s, s_rinv, r, o, k);
          s.ph[(long long)k * s.op + o] = ph;
          slot[pw_phat_off(u.n_ps) + (long long)k * s.op + o] = ph;
        }
      }
    }
    // ---- the unit's last block stamps its PS tiles (after every block's factors) -----------------------------
    __syncthreads();
    if (tid == 0) {
      __threadfence_system();
      const unsigned int old = atomicAdd(&st->cnt_b, 1u);
      s_last = (old == (unsigned int)u.K - 1u) ? 1 : 0;
      if (s_last) { st->cnt_b = 0; __threadfence_system(); }
    }
    __syncthreads();
    if (s_last)
      for (int j = tid; j < u.n_ps; j += PW_THREADS) st_release_sys(reinterpret_cast<int*>(slot) + j, step);
    __syncthreads();
  }
  // ---- the group's push flag -----------------------------------------------------------------------------------
  if (tid == 0) enc_push_flag(a, step);                      // factors and stamps before the counter / push flag
}

// g_hat of 8 columns of row o from this worker's own factors, in the owner's fmaf order (atom order, from 0)
__device__ __forceinline__ void pw_ghat8(const PwScratch& s, int r, int o, const float (&qv)[PW_MAXR][8],
                                         float (&g)[8]) {
  float ph[PW_MAXR];
#pragma unroll
  for (int k = 0; k < PW_MAXR; ++k) ph[k] = k < r ? s.ph[(long long)k * s.op + o] : 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < PW_MAXR; ++k)
      if (k < r) v = fmaf(ph[k], qv[k][j], v);
    g[j] = v;
  }
}

__device__ __forceinline__ void pw_load_q(const PwScratch& s, int r, int c, int C, float (&qv)[PW_MAXR][8]) {
#pragma unroll
  for (int k = 0; k < PW_MAXR; ++k) {
    if (k < r) pw_loadf8(s.q + (long long)k * s.cp, c, C, qv[k]);
    else
#pragma unroll
      for (int j = 0; j < 8; ++j) qv[k][j] = 0.f;
  }
}

// ---- error feedback: e += x - g_hat (pass-A tiles) --------------------------------------------------------------
__global__ void __launch_bounds__(PW_THREADS) v2_powersgd_encode_ef_kernel(const PwArgs a) {
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  if (u.kind != KIND_POWER) return;
  const int r = u.rcap, C = u.cols;
  const PwScratch s = pw_scratch(a.scratch, u);
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
  const bool vec = ((reinterpret_cast<uintptr_t>(gb) & 15) == 0) && (C & 7) == 0;
  for (int c = 8 * threadIdx.x; c < C; c += 8 * PW_THREADS) {
    float qv[PW_MAXR][8];
    pw_load_q(s, r, c, C, qv);
    for (int i = 0; i < t.b; ++i) {
      const int o = t.a + i;
      float x[8], g[8];
      pw_load8(gb + (long long)o * C, c, C, vec, x);
      pw_ghat8(s, r, o, qv, g);
      float* res = a.residual + u.w_off + (long long)o * C + c;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (c + j < C) res[j] += x[j] - g[j];
    }
  }
}

// ---- PS: reconstruct + sum + optimizer ---------------------------------------------------------------------------
template <class A>
__device__ __forceinline__ void ps_powersgd(const A& a) {
  __shared__ float sph[MAX_WORKERS][PW_PS_ROWS][PW_MAXR];   // the counted workers' P_hat rows of one tile
  __shared__ int s_ok, s_bad;
  __shared__ unsigned int s_mask, s_use;
  __shared__ long long s_t_enter, s_t_ready;            // live across the whole launch: kept out of registers
  const int tid = threadIdx.x;
  Ctrl2* ctrl = a.ctrl;
  const int step = ctrl->step;

  ps_wait(a, ctrl, step, s_ok, s_bad, s_mask, s_t_enter, s_t_ready);
  // the counted workers stay inline: as a helper they change this kernel's register allocation
  const bool ok = s_ok != 0;
  const unsigned int wmask = s_mask;
  const bool all_workers = wmask == (a.W >= 32 ? 0xffffffffu : ((1u << a.W) - 1u));
  const OptC c = ps_opt_consts(ctrl, step);
  const float inv_w = all_workers ? a.inv_w : 1.f / (float)max(__popc(wmask), 1);
  const auto [t_begin, t_end] = ps_tile_range(a);
  lw_begin(a);
  for (int ti = t_begin; ok && ti < t_end; ++ti) {
    const Tile2 t = a.tiles[ti];
    const Unit2 u = a.units[t.unit];
    if (u.kind == KIND_VEC) {
      ps_vec_tile(a, c, u, t, wmask, all_workers, inv_w);
      clip_vec_done(a, ti);
      continue;
    }
    if (u.kind == KIND_DENSE16) {
      ps_dense16_tile(a, c, u, t, wmask, inv_w);
      lw_tile_done(a, ti);
      continue;
    }
    if (u.kind != KIND_POWER) continue;
    const int r = u.rcap, C = u.cols, nr = t.b;
    const int op = pw_r4(u.rows), cp = pw_r4(C);
    const int jt = t.a / u.ps_rows;
    const long long phoff = pw_phat_off(u.n_ps), qoff = pw_q_off(u.n_ps, u.rows, r);
    __syncthreads();   // previous tile is done with sph / s_use
    if (tid == 0) s_use = ps_fresh_workers(a, u, jt, wmask, step, s_bad);
    __syncthreads();
    const unsigned int use = s_use;
    for (int idx = tid; idx < MAX_WORKERS * PW_PS_ROWS * PW_MAXR; idx += blockDim.x) {
      const int w = idx / (PW_PS_ROWS * PW_MAXR), i = (idx / PW_MAXR) % PW_PS_ROWS, k = idx % PW_MAXR;
      float v = 0.f;
      if (w < a.W && ((use >> w) & 1u) && i < nr && k < r)
        v = ld_cg_f(a.arenas + (long long)w * a.arena_floats + u.slot_off + phoff + (long long)k * op + t.a + i);
      sph[w][i][k] = v;
    }
    __syncthreads();
    for (int c0 = 8 * tid; c0 < C; c0 += 8 * blockDim.x) {
      float acc[PW_PS_ROWS][8];
#pragma unroll
      for (int i = 0; i < PW_PS_ROWS; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
      for (int w = 0; w < a.W; ++w) {                       // worker order, then atom order
        if (!((use >> w) & 1u)) continue;
        const float* qw = a.arenas + (long long)w * a.arena_floats + u.slot_off + qoff;
        float qv[PW_MAXR][8];
#pragma unroll
        for (int k = 0; k < PW_MAXR; ++k) {
          if (k < r) {
            const float* qk = qw + (long long)k * cp;
            if (c0 + 8 <= C) {
              const float4 x0 = ld_cg_f4(reinterpret_cast<const float4*>(qk + c0));
              const float4 x1 = ld_cg_f4(reinterpret_cast<const float4*>(qk + c0 + 4));
              qv[k][0] = x0.x; qv[k][1] = x0.y; qv[k][2] = x0.z; qv[k][3] = x0.w;
              qv[k][4] = x1.x; qv[k][5] = x1.y; qv[k][6] = x1.z; qv[k][7] = x1.w;
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j) qv[k][j] = (c0 + j < C) ? ld_cg_f(qk + c0 + j) : 0.f;
            }
          }
        }
#pragma unroll
        for (int i = 0; i < PW_PS_ROWS; ++i)
#pragma unroll
          for (int k = 0; k < PW_MAXR; ++k) {
            if (k < r) {
              const float ph = sph[w][i][k];
#pragma unroll
              for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(ph, qv[k][j], acc[i][j]);
            }
          }
      }
      // fused optimizer epilogue + bf16 parameter broadcast
#pragma unroll
      for (int i = 0; i < PW_PS_ROWS; ++i) {
        if (i >= nr) continue;
        const long long e = u.w_off + (long long)(t.a + i) * C + c0;
        if (c0 + 8 <= C && (e & 7) == 0) {
          float g[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) g[j] = acc[i][j] * inv_w;
          update8(a, c, e, g);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (c0 + j < C) update1(a, c, e + j, acc[i][j] * inv_w);
        }
      }
    }
    lw_tile_done(a, ti);
  }

  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, s_bad != 0, s_t_enter, s_t_ready);
}

__global__ void __launch_bounds__(PW_THREADS) v2_ps_powersgd_kernel(const PsArgs2 a) { ps_powersgd(a); }
__global__ void __launch_bounds__(PW_THREADS, 1) v2_ps_powersgd_lw_kernel(const PsArgsLw a) { ps_powersgd(a); }
__global__ void __launch_bounds__(PW_THREADS, 1) v2_ps_powersgd_gather_kernel(const PsArgsGather a) { ps_powersgd(a); }
__global__ void __launch_bounds__(PW_THREADS, 1) v2_ps_powersgd_lion_kernel(const PsArgsLion a) { ps_powersgd(a); }

// ---- --code-stats ------------------------------------------------------------------------------------------------
struct PwStatArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  int tile0;
  const long long* gptr;
  float* scratch;
  const PwState* state;
  double* partials;            // [n_enc_tiles][STAT_PART]
  unsigned int* unit_counters; // [n_coded]
  double* acc;                 // [n_coded][STAT_ACC]
};

__global__ void __launch_bounds__(PW_THREADS) v2_powersgd_code_stats_kernel(const PwStatArgs a) {
  __shared__ double red[2][PW_WARPS];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  if (u.kind != KIND_POWER) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r = u.rcap, C = u.cols;
  const PwScratch s = pw_scratch(a.scratch, u);
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
  const bool vec = ((reinterpret_cast<uintptr_t>(gb) & 15) == 0) && (C & 7) == 0;
  double gsq = 0.0, mse = 0.0;
  for (int c = 8 * tid; c < C; c += 8 * PW_THREADS) {
    float qv[PW_MAXR][8];
    pw_load_q(s, r, c, C, qv);
    for (int i = 0; i < t.b; ++i) {
      float x[8], g[8];
      pw_load8(gb + (long long)(t.a + i) * C, c, C, vec, x);
      pw_ghat8(s, r, t.a + i, qv, g);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (c + j < C) {
          const double xd = (double)x[j], d = xd - (double)g[j];
          gsq = fma(xd, xd, gsq);
          mse = fma(d, d, mse);
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    gsq += __shfl_xor_sync(0xffffffffu, gsq, o);
    mse += __shfl_xor_sync(0xffffffffu, mse, o);
  }
  if (lane == 0) { red[0][warp] = gsq; red[1][warp] = mse; }
  __syncthreads();
  if (tid == 0) {
    double g = 0.0, m = 0.0;
    for (int w = 0; w < PW_WARPS; ++w) { g += red[0][w]; m += red[1][w]; }
    // the non-degenerate columns, counted once per unit
    const double atoms = (t.owner == 0) ? (double)__popc(a.state[u.ts_index].mask) : 0.0;
    stat_store_tile(a, u, g, m, atoms, 0.0, atoms, s_last);
  }
  __syncthreads();
  if (!s_last || tid != 0) return;
  // the unit's sum stays inline: as a helper it changes this kernel's register allocation
  __threadfence();
  double sum[STAT_PART] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < u.n_enc; ++k) {                     // tile order: the same bits on every run
    const double* pk = a.partials + (long long)STAT_PART * (u.enc_tile0 + k);
    for (int f = 0; f < STAT_PART; ++f) sum[f] += __ldcg(pk + f);
  }
  double* acc = a.acc + (long long)STAT_ACC * u.ts_index;
  for (int f = 0; f < STAT_PART; ++f) acc[f] += sum[f];
  acc[5] += sum[4];
  acc[6] += 1.0;
}

// ---- warm-state initialisation (draw 0) -------------------------------------------------------------------------
__global__ void __launch_bounds__(PW_THREADS) v2_powersgd_init_kernel(const Unit2* units, float* scratch,
                                                                      const Ctrl2* ctrl) {
  const Unit2 u = units[blockIdx.x];
  if (u.kind != KIND_POWER) return;
  const PwScratch s = pw_scratch(scratch, u);
  const unsigned long long seed = ctrl->seed;
  for (int k = 0; k < u.rcap; ++k)
    for (int cc = threadIdx.x; cc < s.cp; cc += PW_THREADS)
      s.qw[(long long)k * s.cp + cc] = cc < u.cols ? pw_normal(seed, blockIdx.x, cc, 0, k) : 0.f;
}

extern "C" {

int atomo_v2_powersgd_state_bytes() { return (int)sizeof(PwState); }

void atomo_v2_launch_powersgd_init(const void* units, int n_units, float* scratch, const void* ctrl,
                                   cudaStream_t stream) {
  if (n_units <= 0) return;
  v2_powersgd_init_kernel<<<n_units, PW_THREADS, 0, stream>>>((const Unit2*)units, scratch, (const Ctrl2*)ctrl);
}

void atomo_v2_launch_powersgd_encode(const void* units, const void* enc_tiles, int tile0, int ntiles,
                                     const void* pw_tiles, int pw0, int npw, const long long* gptr, float* scratch,
                                     double* gram, void* state, void* stage, float* const* arena_peer,
                                     int* const* sig_peer, int n_owners, long long arena_floats, int worker, int group,
                                     const void* ctrl, unsigned int* group_counter, long long* tstats,
                                     int final_group, float* residual, cudaStream_t stream) {
  PwArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)enc_tiles + tile0; a.ntiles = ntiles; a.tile0 = tile0;
  a.gptr = gptr; a.scratch = scratch; a.gram = gram; a.state = (PwState*)state; a.stage = (__nv_bfloat16*)stage;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.tstats = tstats; a.final_group = final_group; a.residual = residual;
  if (ntiles > 0) v2_powersgd_encode_a_kernel<<<ntiles, PW_THREADS, 0, stream>>>(a);
  PwArgs b = a;
  b.tiles = (const Tile2*)pw_tiles + pw0; b.ntiles = npw;
  // at least one CTA: it raises the group's push flag even when the group has no PowerSGD unit
  v2_powersgd_encode_b_kernel<<<npw > 0 ? npw : 1, PW_THREADS, 0, stream>>>(b);
  if (residual != nullptr && ntiles > 0) v2_powersgd_encode_ef_kernel<<<ntiles, PW_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_powersgd(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks,
                                 int group, int final_group, int owner, float* master, float* mom, float* sq,
                                 float* sqmax, float* vmom, float* vsq, float* vsqmax, void* wshadow_mc,
                                 void* const* wshadow_peer, float* vparams_local, float* vparams_mc,
                                 float* const* vparams_peer, const float* vgrads_mc, const float* const* vgrads_peer,
                                 const void* const* stage_peer, const float* arenas, long long arena_floats, int* sig,
                                 int* const* sig_peer, void* ctrl, unsigned int* group_counter, long long timeout,
                                 long long* tstats, float inv_w, int grid, cudaStream_t stream) {
  v2_ps_powersgd_kernel<<<ps_grid(grid, ntiles), PW_THREADS, 0, stream>>>(
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, final_group, owner, master, mom, sq, sqmax, vmom, vsq,
              vsqmax, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, vgrads_mc, vgrads_peer,
              stage_peer, arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w));
}

void atomo_v2_launch_powersgd_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                         const long long* gptr, float* scratch, const void* state, double* partials,
                                         unsigned int* unit_counters, double* acc, cudaStream_t stream) {
  if (ntiles <= 0) return;
  PwStatArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr;
  a.scratch = scratch; a.state = (const PwState*)state; a.partials = partials; a.unit_counters = unit_counters;
  a.acc = acc;
  v2_powersgd_code_stats_kernel<<<ntiles, PW_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_powersgd_lw(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLw& a = *static_cast<const PsArgsLw*>(args);
  v2_ps_powersgd_lw_kernel<<<ps_grid(grid, a.ntiles), PW_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_powersgd_gather(const void* args, int grid, cudaStream_t stream) {
  const PsArgsGather& a = *static_cast<const PsArgsGather*>(args);
  v2_ps_powersgd_gather_kernel<<<ps_grid(grid, a.ntiles), PW_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_powersgd_lion(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLion& a = *static_cast<const PsArgsLion*>(args);
  v2_ps_powersgd_lion_kernel<<<ps_grid(grid, a.ntiles), PW_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
