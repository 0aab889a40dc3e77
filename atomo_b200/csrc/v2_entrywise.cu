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
#include "v2_entry_encode.cuh"

namespace atomo {
namespace v2 {

constexpr int EPS_THREADS = 256;

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

// ---- sample + compact + push: entry_encode (v2_entry_encode.cuh) with the sampling keep policy ------------
__global__ void __launch_bounds__(EE_THREADS) v2_entry_encode_kernel(const EEncArgs a) {
  entry_encode<KEEP_SAMPLE, false>(a);
}
// error feedback: the same encode plus the residual epilogue
__global__ void __launch_bounds__(EE_THREADS) v2_entry_encode_ef_kernel(const EEncArgs a) {
  entry_encode<KEEP_SAMPLE, true>(a);
}

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
