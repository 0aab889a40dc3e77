// Entry-wise ATOMO on the overlapped, sharded bf16 engine (sm_90a): worker-side sampling + push of ONE backward
// group, and the owner-side scatter-add + optimizer step.
//
//   v2_entry_stats_kernel    per encode tile, the fp64 L1 norm of the bf16 gradient; the last tile of each unit (unit
//                            counter) adds the partials in tile order into l1[unit], so it has the same bits on
//                            every run.
//   v2_entry_encode_kernel   one CTA per tile (= one destination owner): p_i = min(1, |g_i| * s / L1), element i kept
//                            with probability p_i (Philox keyed by seed / unit / element / step / worker), compacted in
//                            element order by a warp + block scan (no atomics), staged in shared memory and stored
//                            into the owner's arena as 4-byte words, then count / scale and the tile's step stamp;
//                            the last CTA of the launch publishes flag[group][worker] = step on every owner.
//   v2_ps_entry_kernel       one launch per (group, owner): the push wait / --num-aggregate mask of v2_ps_kernel,
//                            fp32 vector tiles, and for entry tiles a scatter-add of the counted workers' entries in
//                            fixed worker order, 1/#counted, then the fused optimizer epilogue and the bf16 broadcast.
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int EE_THREADS = 256;
constexpr int EE_WARPS = EE_THREADS / 32;
constexpr int EE_PER_THREAD = ENTRY_TILE_ELEMS / EE_THREADS;   // 16 consecutive elements per thread
constexpr int EPS_THREADS = 256;
static_assert(EE_PER_THREAD == 16, "a thread loads its elements as two 16-byte chunks");

// The 16 bf16 elements [i0, i0 + 16) of a tile as raw bits, two per word (element 2k in the low half of h[k]); the
// first `rem` of them exist (rem <= 0: none), the rest read as zero.  16-byte loads when the thread's chunk is
// complete and 16-byte aligned (every chunk but the tail of a tensor whose length is not a multiple of 16, unless
// autograd hands over an unaligned gradient).
__device__ __forceinline__ void entry_load16(const __nv_bfloat16* src, int rem, uint32_t (&h)[8]) {
  if (rem >= EE_PER_THREAD && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    const uint4 v0 = __ldg(reinterpret_cast<const uint4*>(src));
    const uint4 v1 = __ldg(reinterpret_cast<const uint4*>(src) + 1);
    h[0] = v0.x; h[1] = v0.y; h[2] = v0.z; h[3] = v0.w; h[4] = v1.x; h[5] = v1.y; h[6] = v1.z; h[7] = v1.w;
    return;
  }
  const unsigned short* s16 = reinterpret_cast<const unsigned short*>(src);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t lo = (2 * k < rem) ? (uint32_t)s16[2 * k] : 0u;
    const uint32_t hi = (2 * k + 1 < rem) ? (uint32_t)s16[2 * k + 1] : 0u;
    h[k] = lo | (hi << 16);
  }
}
__device__ __forceinline__ uint32_t bf16_bits(const uint32_t (&h)[8], int i) {
  return (i & 1) ? (h[i >> 1] >> 16) : (h[i >> 1] & 0xffffu);
}

// ---- L1 norm: per-tile fp64 partials, combined in tile order by the unit's last tile ------------------------
struct EStatArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  int tile0;                   // global index of tiles[0] (partials are indexed by global encode tile)
  const long long* gptr;
  double* partials;            // [n_enc_tiles]
  unsigned int* unit_counters; // [n_entry_units]
  double* l1;                  // [n_entry_units]
  long long* tstats;
  int group;
};

__global__ void __launch_bounds__(EE_THREADS) v2_entry_stats_kernel(const EStatArgs a) {
  __shared__ double red[EE_WARPS];
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();
  const int i0 = tid * EE_PER_THREAD;
  uint32_t h[8];
  entry_load16(reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a + i0, t.b - i0, h);
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < EE_PER_THREAD; ++i) s += (double)fabsf(__uint_as_float(bf16_bits(h, i) << 16));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (tid == 0) {
    double ts = 0.0;
    for (int w = 0; w < EE_WARPS; ++w) ts += red[w];
    a.partials[a.tile0 + blockIdx.x] = ts;
    __threadfence();
    const unsigned int old = atomicAdd(&a.unit_counters[u.ts_index], 1u);
    if (old == (unsigned int)u.n_enc - 1u) {
      a.unit_counters[u.ts_index] = 0;
      __threadfence();
      double L1 = 0.0;
      for (int k = 0; k < u.n_enc; ++k) L1 += __ldcg(a.partials + u.enc_tile0 + k);   // fixed order
      a.l1[u.ts_index] = L1;
    }
  }
}

// ---- sample + compact + push -------------------------------------------------------------------------------
struct EEncArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  const long long* gptr;       // gradient base pointers (bf16), one per weight tensor
  const double* l1;            // per entry unit (v2_entry_stats_kernel)
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
  float* residual;             // error feedback (v2_feedback.cu): fp32 residual indexed like wshadow, or nullptr
};

// Error feedback: what element x of A is owed after this push, x - g_hat (the owner's decode of the tile)
__device__ __forceinline__ float entry_residual(uint32_t bits, uint32_t kept, uint32_t exact, float scale) {
  const float x = __uint_as_float(bits << 16);
  return kept ? (exact ? 0.f : x - copysignf(scale, x)) : x;
}

// The uniform of element e of a unit is word (e & 3) of Philox(seed', counter = (e >> 2, unit, step, worker)):
// one Philox call serves 4 consecutive elements.  The seed differs from the QSGD rounding's.
__device__ __forceinline__ void entry_philox(const EEncArgs& a, int unit, long long e, int step, uint32_t (&r4)[4]) {
  Philox::gen(a.ctrl->seed ^ 0xd1b54a32d192ed03ULL, (uint32_t)(e >> 2), (uint32_t)unit, (uint32_t)step,
              (uint32_t)a.worker, r4);
}

template <bool EF>
__device__ __forceinline__ void entry_encode(const EEncArgs& a) {
  __shared__ __align__(16) uint32_t ent[ENTRY_TILE_ELEMS];
  __shared__ int wsum[EE_WARPS];
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int step = a.ctrl->step;
  const int jt = t.owner;                                   // encode tiles: index of the tile inside its unit
  const int owner = (u.own0 + jt) % a.n_owners;
  float* slot = a.arena_peer[owner] + (long long)a.worker * a.arena_floats + u.slot_off;
  // k = s / L1 and the value of a non-clamped entry, L1 / s, from the fp64 norm.  L1 == 0 (or NaN) keeps nothing.
  const double L1 = a.l1[u.ts_index], s = (double)u.budget;
  const bool live = L1 > 0.0;
  const float k = live ? (float)(s / L1) : 0.f;
  const float scale = live ? (float)(L1 / s) : 0.f;

  const int i0 = tid * EE_PER_THREAD;
  const int n = t.b - i0;                                   // elements of this thread (<= 0: none, >= 16: 16)
  uint32_t h[8];
  entry_load16(reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a + i0, n, h);
  const long long e0 = (long long)t.a + i0;                 // element index inside the unit (a multiple of 16)
  uint32_t keep = 0, exact = 0;
  uint32_t r4[4];
#pragma unroll
  for (int i = 0; i < EE_PER_THREAD; ++i) {
    if (i < n && live) {
      float uu;
      if (a.ext_uniforms != nullptr) {
        uu = a.ext_uniforms[u.w_off + e0 + i];
      } else {
        if ((i & 3) == 0) entry_philox(a, t.unit, e0 + i, step, r4);
        uu = Philox::to_uniform(r4[i & 3]);
      }
      const float p = fabsf(__uint_as_float(bf16_bits(h, i) << 16)) * k;   // clamped to 1 below: u < 1 <= p
      if (uu < p) keep |= 1u << i;
      if (p >= 1.f) exact |= 1u << i;
    }
  }
  if (EF && n > 0) {
    float* ep = a.residual + u.w_off + e0;                   // 64-byte aligned: w_off % 64 == 0, e0 % 16 == 0
    if (n >= EE_PER_THREAD) {
#pragma unroll
      for (int j = 0; j < EE_PER_THREAD / 4; ++j) {
        float4 v = reinterpret_cast<const float4*>(ep)[j];
        const int i = 4 * j;
        v.x += entry_residual(bf16_bits(h, i), (keep >> i) & 1u, (exact >> i) & 1u, scale);
        v.y += entry_residual(bf16_bits(h, i + 1), (keep >> (i + 1)) & 1u, (exact >> (i + 1)) & 1u, scale);
        v.z += entry_residual(bf16_bits(h, i + 2), (keep >> (i + 2)) & 1u, (exact >> (i + 2)) & 1u, scale);
        v.w += entry_residual(bf16_bits(h, i + 3), (keep >> (i + 3)) & 1u, (exact >> (i + 3)) & 1u, scale);
        reinterpret_cast<float4*>(ep)[j] = v;
      }
    } else {
      for (int i = 0; i < n; ++i) ep[i] += entry_residual(bf16_bits(h, i), (keep >> i) & 1u, (exact >> i) & 1u, scale);
    }
  }

  // ---- compaction in element order: warp scan of the per-thread counts, then the warp totals -------------------
  const int cnt = __popc(keep);
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  int pos = incl - cnt, total = 0;
#pragma unroll
  for (int w = 0; w < EE_WARPS; ++w) {
    const int v = wsum[w];
    if (w < warp) pos += v;
    total += v;
  }
#pragma unroll
  for (int i = 0; i < EE_PER_THREAD; ++i)
    if ((keep >> i) & 1u)
      ent[pos++] = (uint32_t)(i0 + i) | (((exact >> i) & 1u) ? ENTRY_FLAG_EXACT : 0u) | (bf16_bits(h, i) << 16);
  if (tid < ((total + 3) & ~3) - total) ent[total + tid] = 0u;   // the last 16-byte store carries no stale words
  __syncthreads();

  uint4* dst = reinterpret_cast<uint4*>(slot + entry_words_off(u.n_ps, jt, u.ps_rows));
  for (int v = tid; v < (total + 3) >> 2; v += EE_THREADS) dst[v] = *reinterpret_cast<const uint4*>(&ent[4 * v]);
  int* hdr = reinterpret_cast<int*>(slot + entry_hdr_off(jt));
  if (tid == 0) {
    hdr[1] = total;
    hdr[2] = __float_as_int(scale);
    hdr[3] = 0;
  }

  // ---- the tile's step stamp (after its entries, count and scale), then the group's push flag -----------------
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();                                   // entries + count + scale before the stamp
    st_release_sys(hdr, step);
    __threadfence_system();                                   // the stamp before the counter (and so the push flag)
    const unsigned int old = atomicAdd(a.group_counter, 1u);
    if (old == gridDim.x - 1) {
      *a.group_counter = 0;
      __threadfence_system();
      for (int o = 0; o < a.n_owners; ++o)
        st_release_sys(a.sig_peer[o] + SIG_PUSH + a.group * MAX_WORKERS + a.worker, step);
      if (a.tstats != nullptr) {
        const long long now = globaltimer_ns();
        a.tstats[5] += now - a.tstats[9 + a.group];      // stats + encode of this group
        if (a.final_group) a.tstats[8] += now - a.tstats[6];          // step start -> last push published
      }
    }
  }
}

__global__ void __launch_bounds__(EE_THREADS) v2_entry_encode_kernel(const EEncArgs a) { entry_encode<false>(a); }
// error feedback: the same encode plus the residual epilogue
__global__ void __launch_bounds__(EE_THREADS) v2_entry_encode_ef_kernel(const EEncArgs a) { entry_encode<true>(a); }

// ---- PS: scatter-add + optimizer --------------------------------------------------------------------------
__global__ void __launch_bounds__(EPS_THREADS) v2_ps_entry_kernel(const PsArgs2 a) {
  __shared__ __align__(16) float OUT[ENTRY_TILE_ELEMS];   // summed entries of one tile, physical element order
  __shared__ int s_ok, s_bad;
  __shared__ unsigned int s_mask, s_use;
  const int tid = threadIdx.x;
  Ctrl2* ctrl = a.ctrl;
  const int step = ctrl->step;

  long long t_enter = 0, t_ready = 0;
  if (tid == 0) {
    t_enter = globaltimer_ns();
    unsigned int mask;
    const bool ok = ps_wait_pushes(a, ctrl, step, mask);
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
  const OptC c = ps_opt_consts(ctrl, step);
  const float inv_w = all_workers ? a.inv_w : 1.f / (float)max(__popc(wmask), 1);

  const int per_cta = (a.ntiles + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta;
  const int t_end = min(a.ntiles, t_begin + per_cta);
  for (int ti = t_begin; ok && ti < t_end; ++ti) {
    const Tile2 t = a.tiles[ti];
    const Unit2 u = a.units[t.unit];
    if (u.kind == KIND_VEC) {
      ps_vec_tile(a, c, u, t, wmask, all_workers, inv_w);
      continue;
    }
    if (u.kind != KIND_ENTRY) continue;
    const int jt = t.a / u.ps_rows;
    __syncthreads();   // previous tile is done with OUT / s_use
    if (tid == 0) {
      unsigned int use = 0;
      for (int w = 0; w < a.W; ++w) {
        if (!((wmask >> w) & 1u)) continue;
        const int* hdr = reinterpret_cast<const int*>(a.arenas + (long long)w * a.arena_floats + u.slot_off +
                                                      entry_hdr_off(jt));
        if (ld_cg_i(hdr) == step) use |= 1u << w;
        else s_bad = 1;                                  // stale slot: a push of another step
      }
      s_use = use;
    }
    for (int i = tid; i < t.b; i += blockDim.x) OUT[i] = 0.f;
    __syncthreads();
    const unsigned int use = s_use;
    // worker by worker in worker order: one worker's offsets are distinct, so its adds do not race, and every
    // element receives its terms in the same order on every run
    for (int w = 0; w < a.W; ++w) {
      if (!((use >> w) & 1u)) continue;
      const float* sw = a.arenas + (long long)w * a.arena_floats + u.slot_off;
      const int* hdr = reinterpret_cast<const int*>(sw + entry_hdr_off(jt));
      const int cnt = min(ld_cg_i(hdr + 1), t.b);
      const float scale = __int_as_float(ld_cg_i(hdr + 2));
      const uint32_t* wd = reinterpret_cast<const uint32_t*>(sw + entry_words_off(u.n_ps, jt, u.ps_rows));
      for (int v = tid; v < (cnt + 3) >> 2; v += blockDim.x) {
        const uint4 q = ld_cg_u4(wd + 4 * v);
        const uint32_t e4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (4 * v + j < cnt) {
            const uint32_t e = e4[j];
            const float g = __uint_as_float(e & 0xffff0000u);
            const float val = (e & ENTRY_FLAG_EXACT) ? g : copysignf(scale, g);
            OUT[e & 0xfffu] = __fadd_rn(OUT[e & 0xfffu], val);
          }
        }
      }
      __syncthreads();
    }
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
  }

  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, s_bad != 0, t_enter, t_ready);
}

extern "C" {

void atomo_v2_launch_entry_stats(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 double* partials, unsigned int* unit_counters, double* l1, long long* tstats,
                                 int group, cudaStream_t stream) {
  if (ntiles <= 0) return;
  EStatArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr;
  a.partials = partials; a.unit_counters = unit_counters; a.l1 = l1; a.tstats = tstats; a.group = group;
  v2_entry_stats_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_entry_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                  const double* l1, float* const* arena_peer, int* const* sig_peer, int n_owners,
                                  long long arena_floats, int worker, int group, const void* ctrl,
                                  unsigned int* group_counter, const float* ext_uniforms, long long* tstats,
                                  int final_group, float* residual, cudaStream_t stream) {
  if (ntiles <= 0) return;
  EEncArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr; a.l1 = l1;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.ext_uniforms = ext_uniforms; a.tstats = tstats; a.final_group = final_group; a.residual = residual;
  if (residual != nullptr) v2_entry_encode_ef_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a);
  else v2_entry_encode_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_entry(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks,
                              int group, int final_group, int owner, float* master, float* mom, float* sq,
                              float* sqmax, float* vmom, float* vsq, float* vsqmax, void* wshadow_mc,
                              void* const* wshadow_peer, float* vparams_local, float* vparams_mc,
                              float* const* vparams_peer, const float* vgrads_mc, const float* const* vgrads_peer,
                              const float* arenas, long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                              unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                              cudaStream_t stream) {
  PsArgs2 a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.ntiles = ntiles; a.W = W; a.nranks = nranks;
  a.group = group; a.final_group = final_group; a.owner = owner; a.master = master; a.mom = mom; a.sq = sq;
  a.sqmax = sqmax; a.vmom = vmom; a.vsq = vsq; a.vsqmax = vsqmax; a.wshadow_mc = (__nv_bfloat16*)wshadow_mc;
  a.wshadow_peer = (__nv_bfloat16* const*)wshadow_peer; a.vparams_local = vparams_local; a.vparams_mc = vparams_mc;
  a.vparams_peer = vparams_peer; a.vgrads_mc = vgrads_mc; a.vgrads_peer = vgrads_peer; a.stage_peer = nullptr;
  a.arenas = arenas; a.arena_floats = arena_floats; a.sig = sig; a.sig_peer = sig_peer; a.ctrl = (Ctrl2*)ctrl;
  a.group_counter = group_counter; a.timeout = timeout; a.tstats = tstats; a.inv_w = inv_w;
  if (grid < 1) grid = 1;
  if (ntiles > 0 && grid > ntiles) grid = ntiles;
  v2_ps_entry_kernel<<<grid, EPS_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
