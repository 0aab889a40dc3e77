// QSGD / TernGrad on the overlapped, sharded bf16 engine (sm_90a): worker-side quantize + push of ONE backward
// group, and the owner-side decode + optimizer step.
//
//   v2_qsgd_stats_kernel   TernGrad only: per encode tile, sum and sum of squares of the bf16 gradient (fp64);
//                          the last tile of each unit (unit counter) combines the partials in tile order into
//                          clip[unit] = 2.5 * population std of the whole tensor.
//   v2_qsgd_encode_kernel  one CTA per PS tile (= one destination owner), one warp per bucket: bf16 gradient read
//                          in place through the pointer table with 16-byte loads, fp32 norm (QSGD: L2; TernGrad:
//                          L-inf after the clip), unbiased stochastic rounding (round up with probability frac,
//                          Philox keyed by seed / unit / element / step / worker), section-major packing exactly as
//                          codings/qsgd.py, words + norms stored into the owner's arena, then the tile's step stamp;
//                          the last CTA of the launch publishes flag[group][worker] = step on every owner.
//   v2_ps_qsgd_kernel      one launch per (group, owner): the push wait / --num-aggregate mask of v2_ps_kernel,
//                          fp32 vector tiles, and for QSGD tiles the decode + sum of the counted workers' buckets in
//                          fixed worker order (TernGrad: every worker scaled by the max norm over the counted
//                          workers), 1/#counted, then the fused optimizer epilogue and the bf16 broadcast.
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int QE_THREADS = 256;
constexpr int QE_WARPS = QE_THREADS / 32;
constexpr int QE_MAX_BUCKET = 1024;
constexpr int QPS_THREADS = 256;
constexpr int QPS_TILE_ELEMS = 4096;

struct QEncArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  const long long* gptr;       // gradient base pointers (bf16), one per weight tensor
  const float* clip;           // TernGrad: per QSGD unit clip limit (v2_qsgd_stats_kernel), else unused
  float* const* arena_peer;    // [n_owners] arena base inside each owner
  int* const* sig_peer;        // [n_owners] signal region base of each owner
  int n_owners;
  long long arena_floats;
  int worker;
  int group;
  const Ctrl2* ctrl;
  unsigned int* group_counter;
  const float* ext_uniforms;   // tests: uniforms indexed like wshadow, replacing Philox
  long long* tstats;
  int final_group;
  int stamp_start;             // 1: this launch stamps the group's encode start (no stats launch before it)
  float* residual;             // error feedback (v2_feedback.cu, QSGD only): fp32 residual like wshadow, or nullptr
};

__device__ __forceinline__ void bf16x8(const uint4 v, float (&x)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { x[2 * i] = bf16_lo(w[i]); x[2 * i + 1] = bf16_hi(w[i]); }
}

// The uniform of element e of a unit is word (e & 3) of Philox(seed', counter = (e >> 2, unit, step, worker)):
// one Philox call serves 4 consecutive elements.
__device__ __forceinline__ void qsgd_philox(const QEncArgs& a, int unit, long long e, int step, uint32_t (&r4)[4]) {
  Philox::gen(a.ctrl->seed ^ 0x9e3779b97f4a7c15ULL, (uint32_t)(e >> 2), (uint32_t)unit, (uint32_t)step,
              (uint32_t)a.worker, r4);
}
__device__ __forceinline__ float pick4(const uint32_t (&r4)[4], int k) {
  return Philox::to_uniform(k == 0 ? r4[0] : k == 1 ? r4[1] : k == 2 ? r4[2] : r4[3]);
}
__device__ __forceinline__ float qsgd_uniform(const QEncArgs& a, const Unit2& u, int unit, long long e, int step) {
  if (a.ext_uniforms != nullptr) return a.ext_uniforms[u.w_off + e];
  uint32_t r4[4];
  qsgd_philox(a, unit, e, step, r4);
  return pick4(r4, (int)(e & 3));
}

__device__ __forceinline__ unsigned short qsgd_code(float x, float inv, int levels, int q, float u) {
  const float av = fminf(fabsf(x) * inv, (float)levels);
  const float lo = floorf(av);
  const int xi = min((int)lo + (u < av - lo ? 1 : 0), levels);
  const int sgn = (x > 0.f) ? 2 : (x < 0.f ? 0 : 1);
  return (unsigned short)((sgn << q) | xi);
}

// The owner's decode of one code (v2_ps_qsgd_kernel): sign * level * (norm / levels), with the same roundings
__device__ __forceinline__ float qsgd_dequant(uint32_t cd, int q, int levels, float scale) {
  const float xi = (float)(int)(cd & (uint32_t)levels);
  const float sg = (float)((int)(cd >> q) & 3) - 1.f;
  return __fmul_rn(sg * xi, scale);
}

template <bool EF>
__device__ __forceinline__ void qsgd_encode(const QEncArgs& a) {
  __shared__ __align__(16) unsigned short codes[QE_WARPS][QE_MAX_BUCKET];
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr && a.stamp_start) a.tstats[9 + a.group] = globaltimer_ns();
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
  const int bucket = u.K, q = u.I, L = u.cols;
  const int levels = (1 << q) - 1, E = 64 / (2 + q);
  const bool tern = u.rs != 0;
  const float clip = tern ? a.clip[u.ts_index] : 0.f;
  const int step = a.ctrl->step;
  const int jt = t.owner;                                   // encode tiles: index of the tile inside its unit
  const int owner = (u.own0 + jt) % a.n_owners;
  float* slot = a.arena_peer[owner] + (long long)a.worker * a.arena_floats + u.slot_off;
  float* norms = slot + qsgd_norms_off(u.n_ps);
  unsigned long long* words = reinterpret_cast<unsigned long long*>(slot + qsgd_words_off(u.n_ps, u.rows));
  const int kb0 = t.a / bucket, nbt = (t.b + bucket - 1) / bucket;

  for (int kb = warp; kb < nbt; kb += QE_WARPS) {
    const long long bk = kb0 + kb;
    const long long e0 = bk * bucket;
    const int blen = (int)min((long long)bucket, (long long)u.numel - e0);
    const __nv_bfloat16* src = gb + e0;
    // 16-byte loads when the bucket starts on an 8-element boundary of the tensor and of memory (every bucket but
    // the single, odd-sized bucket of a tensor smaller than bucket_size starts on one)
    const int nch = (((reinterpret_cast<uintptr_t>(src) & 15) | (e0 & 7)) == 0) ? (blen >> 3) : 0;
    // pass 1: norm (QSGD: L2; TernGrad: L-inf of the clipped values)
    float acc = 0.f;
    for (int c = lane; c < nch; c += 32) {
      float x[8];
      bf16x8(__ldg(reinterpret_cast<const uint4*>(src) + c), x);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (tern) acc = fmaxf(acc, fabsf(clip > 0.f ? fminf(fmaxf(x[i], -clip), clip) : x[i]));
        else acc = fmaf(x[i], x[i], acc);
      }
    }
    for (int i = (nch << 3) + lane; i < blen; i += 32) {
      float x = __bfloat162float(src[i]);
      if (tern) acc = fmaxf(acc, fabsf(clip > 0.f ? fminf(fmaxf(x, -clip), clip) : x));
      else acc = fmaf(x, x, acc);
    }
    const float nrm = tern ? warp_max(acc) : sqrtf(warp_sum(acc));
    const float inv = nrm > 0.f ? (float)levels / nrm : 0.f;
    const float dq = EF ? __fdiv_rn(nrm, (float)levels) : 0.f;   // error feedback: the owner's scale of the bucket
    float* res = EF ? a.residual + u.w_off + e0 : nullptr;
    // pass 2: stochastic rounding into codes (the bucket is L1 resident from pass 1)
    for (int c = lane; c < nch; c += 32) {
      float x[8];
      bf16x8(__ldg(reinterpret_cast<const uint4*>(src) + c), x);
      uint32_t r4[4];
      uint32_t packed[4];    // the lane's 8 codes go to shared memory as ONE 16-byte store (no bank conflicts)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float v = (tern && clip > 0.f) ? fminf(fmaxf(x[i], -clip), clip) : x[i];
        const int el = 8 * c + i;
        const long long e = e0 + el;
        float uu;
        if (a.ext_uniforms != nullptr) {
          uu = a.ext_uniforms[u.w_off + e];
        } else {
          if ((i & 3) == 0) qsgd_philox(a, t.unit, e, step, r4);     // e0 % 8 == 0: e & 3 == i & 3
          uu = Philox::to_uniform(r4[i & 3]);
        }
        const uint32_t cd = qsgd_code(v, inv, levels, q, uu);
        if (i & 1) packed[i >> 1] |= cd << 16;
        else packed[i >> 1] = cd;
      }
      *reinterpret_cast<uint4*>(&codes[warp][8 * c]) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
      if (EF) {                      // e += x - g_hat; 32-byte aligned (w_off % 64 == 0, e0 % 8 == 0)
        float4* rp = reinterpret_cast<float4*>(res + 8 * c);
        float4 r0 = rp[0], r1 = rp[1];
        r0.x += x[0] - qsgd_dequant(packed[0] & 0xffffu, q, levels, dq);
        r0.y += x[1] - qsgd_dequant(packed[0] >> 16, q, levels, dq);
        r0.z += x[2] - qsgd_dequant(packed[1] & 0xffffu, q, levels, dq);
        r0.w += x[3] - qsgd_dequant(packed[1] >> 16, q, levels, dq);
        r1.x += x[4] - qsgd_dequant(packed[2] & 0xffffu, q, levels, dq);
        r1.y += x[5] - qsgd_dequant(packed[2] >> 16, q, levels, dq);
        r1.z += x[6] - qsgd_dequant(packed[3] & 0xffffu, q, levels, dq);
        r1.w += x[7] - qsgd_dequant(packed[3] >> 16, q, levels, dq);
        rp[0] = r0; rp[1] = r1;
      }
    }
    for (int i = (nch << 3) + lane; i < blen; i += 32) {
      float x = __bfloat162float(src[i]);
      if (tern && clip > 0.f) x = fminf(fmaxf(x, -clip), clip);
      const unsigned short cd = qsgd_code(x, inv, levels, q, qsgd_uniform(a, u, t.unit, e0 + i, step));
      codes[warp][i] = cd;
      if (EF) res[i] += x - qsgd_dequant(cd, q, levels, dq);
    }
    __syncwarp();
    // section-major packing: word j holds elements j, j+L, j+2L, ... (section 0 in the MSBs); padding (zero tail of
    // the last bucket and the slack of the last word) encodes sign 0, level 0 = 1 << q
    for (int j = lane; j < L; j += 32) {
      unsigned long long w = 0ULL;
      for (int s = 0; s < E; ++s) {
        const int i = s * L + j;
        const unsigned long long c = (i < blen) ? (unsigned long long)codes[warp][i] : (1ULL << q);
        w = (w << (2 + q)) | c;
      }
      words[bk * L + j] = w;
    }
    if (lane == 0) norms[bk] = nrm;
    __syncwarp();
  }

  // ---- the tile's step stamp (after its words and norms), then the group's push flag ----------------------
  __syncthreads();
  if (tid == 0) {
    enc_stamp(reinterpret_cast<int*>(slot), jt, step);
    enc_push_flag(a, step);
  }
}

__global__ void __launch_bounds__(QE_THREADS) v2_qsgd_encode_kernel(const QEncArgs a) { qsgd_encode<false>(a); }
// error feedback: the same encode plus the residual epilogue
__global__ void __launch_bounds__(QE_THREADS) v2_qsgd_encode_ef_kernel(const QEncArgs a) { qsgd_encode<true>(a); }

// ---- TernGrad clip: per-tile (sum, sum of squares) in fp64, combined in tile order by the unit's last tile ----
struct QStatArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  int tile0;                   // global index of tiles[0] (partials are indexed by global encode tile)
  const long long* gptr;
  double* partials;            // [n_enc_tiles][2]
  unsigned int* unit_counters; // [n_qsgd_units]
  float* clip;                 // [n_qsgd_units]
  long long* tstats;
  int group;
};

__global__ void __launch_bounds__(QE_THREADS) v2_qsgd_stats_kernel(const QStatArgs a) {
  __shared__ double red[2][QE_WARPS];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();
  const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a;
  const int nch = ((reinterpret_cast<uintptr_t>(src) & 15) == 0) ? (t.b >> 3) : 0;
  double s = 0.0, ss = 0.0;
  for (int c = tid; c < nch; c += blockDim.x) {
    float x[8];
    bf16x8(__ldg(reinterpret_cast<const uint4*>(src) + c), x);
#pragma unroll
    for (int i = 0; i < 8; ++i) { s += (double)x[i]; ss = fma((double)x[i], (double)x[i], ss); }
  }
  for (int i = (nch << 3) + tid; i < t.b; i += blockDim.x) {
    const double x = (double)__bfloat162float(src[i]);
    s += x; ss = fma(x, x, ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  if (lane == 0) { red[0][warp] = s; red[1][warp] = ss; }
  __syncthreads();
  if (tid == 0) {
    double ts = 0.0, tss = 0.0;
    for (int w = 0; w < QE_WARPS; ++w) { ts += red[0][w]; tss += red[1][w]; }
    double* p = a.partials + 2LL * (a.tile0 + blockIdx.x);
    p[0] = ts; p[1] = tss;
    __threadfence();
    const unsigned int old = atomicAdd(&a.unit_counters[u.ts_index], 1u);
    s_last = (old == (unsigned int)u.n_enc - 1u) ? 1 : 0;
    if (s_last) {
      a.unit_counters[u.ts_index] = 0;
      __threadfence();
      double S = 0.0, SS = 0.0;
      for (int k = 0; k < u.n_enc; ++k) {           // fixed order: the clip has the same bits on every run
        const double* pk = a.partials + 2LL * (u.enc_tile0 + k);
        S += __ldcg(pk); SS += __ldcg(pk + 1);
      }
      const double n = (double)u.numel, mean = S / n;
      const double var = fmax(SS / n - mean * mean, 0.0);
      a.clip[u.ts_index] = u.numel > 1 ? (float)(2.5 * sqrt(var)) : 0.f;
    }
  }
}

// ---- PS: decode + sum + optimizer --------------------------------------------------------------------------
template <class A>
__device__ __forceinline__ void ps_qsgd(const A& a) {
  __shared__ __align__(16) float OUT[QPS_TILE_ELEMS];   // summed decodes of one tile, physical element order
  __shared__ int s_ok, s_bad;
  __shared__ unsigned int s_mask, s_use;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  Ctrl2* ctrl = a.ctrl;
  const int step = ctrl->step;

  long long t_enter = 0, t_ready = 0;
  ps_wait(a, ctrl, step, s_ok, s_bad, s_mask, t_enter, t_ready);
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
    if (u.kind != KIND_QSGD) continue;
    const int bucket = u.K, q = u.I, L = u.cols;
    const int levels = (1 << q) - 1, E = 64 / (2 + q);
    const unsigned long long cmask = (1ULL << (2 + q)) - 1ULL;
    const bool tern = u.rs != 0;
    const int kb0 = t.a / bucket, nbt = (t.b + bucket - 1) / bucket;
    const int jt = kb0 / u.cs;
    const long long noff = qsgd_norms_off(u.n_ps), woff = qsgd_words_off(u.n_ps, u.rows);
    __syncthreads();   // previous tile is done with OUT / s_use
    if (tid == 0) s_use = ps_fresh_workers(a, u, jt, wmask, step, s_bad);
    for (int i = tid; i < t.b; i += blockDim.x) OUT[i] = 0.f;
    __syncthreads();
    const unsigned int use = s_use;
    // one warp per bucket; lane j owns the elements of words j, j+32, ... so the per-element sum over workers
    // runs in worker order without any cross-lane interaction
    for (int kb = warp; kb < nbt; kb += blockDim.x >> 5) {
      const long long bk = kb0 + kb;
      const int blen = min(bucket, t.b - kb * bucket);
      float nmax = 0.f;
      if (tern)
        for (int w = 0; w < a.W; ++w)
          if ((use >> w) & 1u) nmax = fmaxf(nmax, ld_cg_f(a.arenas + (long long)w * a.arena_floats + u.slot_off + noff + bk));
      float* o = OUT + kb * bucket;
      for (int w = 0; w < a.W; ++w) {
        if (!((use >> w) & 1u)) continue;
        const float* sw = a.arenas + (long long)w * a.arena_floats + u.slot_off;
        // IEEE division (not the fast-math approximation): the same scale as codings.qsgd's norms / s, so that
        // decodes that cancel across workers cancel exactly here too
        const float scale = __fdiv_rn(tern ? nmax : ld_cg_f(sw + noff + bk), (float)levels);
        const unsigned long long* wd = reinterpret_cast<const unsigned long long*>(sw + woff) + bk * L;
        for (int j = lane; j < L; j += 32) {
          unsigned long long v;
          asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(v) : "l"(wd + j));
          for (int s = 0; s < E; ++s) {
            const int i = s * L + j;
            if (i < blen) {
              const unsigned long long cd = (v >> ((E - 1 - s) * (2 + q))) & cmask;
              const float xi = (float)(int)(cd & (unsigned long long)levels);
              const float sg = (float)((int)(cd >> q) & 3) - 1.f;
              o[i] = __fadd_rn(o[i], __fmul_rn(sg * xi, scale));   // no FMA contraction: the coder's roundings
            }
          }
        }
      }
    }
    __syncthreads();
    // fused optimizer epilogue + bf16 parameter broadcast
    const long long e0 = u.w_off + t.a;
    const int nvec = ((e0 & 7) == 0) ? (t.b >> 3) : 0;
    for (int v = tid; v < nvec; v += blockDim.x) {
      const float4 g0 = *reinterpret_cast<const float4*>(&OUT[8 * v]);
      const float4 g1 = *reinterpret_cast<const float4*>(&OUT[8 * v + 4]);
      const float g[8] = {g0.x * inv_w, g0.y * inv_w, g0.z * inv_w, g0.w * inv_w,
                          g1.x * inv_w, g1.y * inv_w, g1.z * inv_w, g1.w * inv_w};
      update8(a, c, e0 + 8LL * v, g);
    }
    for (int i = (nvec << 3) + tid; i < t.b; i += blockDim.x) update1(a, c, e0 + i, OUT[i] * inv_w);
    lw_tile_done(a, ti);
  }

  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, s_bad != 0, t_enter, t_ready);
}

__global__ void __launch_bounds__(QPS_THREADS) v2_ps_qsgd_kernel(const PsArgs2 a) { ps_qsgd(a); }
__global__ void __launch_bounds__(QPS_THREADS, 1) v2_ps_qsgd_lw_kernel(const PsArgsLw a) { ps_qsgd(a); }
__global__ void __launch_bounds__(QPS_THREADS, 1) v2_ps_qsgd_gather_kernel(const PsArgsGather a) { ps_qsgd(a); }
__global__ void __launch_bounds__(QPS_THREADS, 1) v2_ps_qsgd_lion_kernel(const PsArgsLion a) { ps_qsgd(a); }

extern "C" {

void atomo_v2_launch_qsgd_stats(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                double* partials, unsigned int* unit_counters, float* clip, long long* tstats,
                                int group, cudaStream_t stream) {
  if (ntiles <= 0) return;
  QStatArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr;
  a.partials = partials; a.unit_counters = unit_counters; a.clip = clip; a.tstats = tstats; a.group = group;
  v2_qsgd_stats_kernel<<<ntiles, QE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_qsgd_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 const float* clip, float* const* arena_peer, int* const* sig_peer, int n_owners,
                                 long long arena_floats, int worker, int group, const void* ctrl,
                                 unsigned int* group_counter, const float* ext_uniforms, long long* tstats,
                                 int final_group, int stamp_start, float* residual, cudaStream_t stream) {
  if (ntiles <= 0) return;
  QEncArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr; a.clip = clip;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.ext_uniforms = ext_uniforms; a.tstats = tstats; a.final_group = final_group; a.stamp_start = stamp_start;
  a.residual = residual;
  if (residual != nullptr) v2_qsgd_encode_ef_kernel<<<ntiles, QE_THREADS, 0, stream>>>(a);
  else v2_qsgd_encode_kernel<<<ntiles, QE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_qsgd(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                             int final_group, int owner, float* master, float* mom, float* sq, float* sqmax,
                             float* vmom, float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer,
                             float* vparams_local, float* vparams_mc, float* const* vparams_peer,
                             const float* vgrads_mc, const float* const* vgrads_peer, const float* arenas,
                             long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                             unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                             cudaStream_t stream) {
  v2_ps_qsgd_kernel<<<ps_grid(grid, ntiles), QPS_THREADS, 0, stream>>>(
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, final_group, owner, master, mom, sq, sqmax, vmom, vsq,
              vsqmax, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, vgrads_mc, vgrads_peer,
              nullptr, arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w));
}

void atomo_v2_launch_ps_qsgd_lw(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLw& a = *static_cast<const PsArgsLw*>(args);
  v2_ps_qsgd_lw_kernel<<<ps_grid(grid, a.ntiles), QPS_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_qsgd_gather(const void* args, int grid, cudaStream_t stream) {
  const PsArgsGather& a = *static_cast<const PsArgsGather*>(args);
  v2_ps_qsgd_gather_kernel<<<ps_grid(grid, a.ntiles), QPS_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_qsgd_lion(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLion& a = *static_cast<const PsArgsLion*>(args);
  v2_ps_qsgd_lion_kernel<<<ps_grid(grid, a.ntiles), QPS_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
