// Scaled sign (EF-SignSGD) on the overlapped, sharded bf16 engine (sm_90a): worker-side encode + push of ONE backward
// group, the owner-side decode + optimizer step, and --code-stats.  The oracle is codings/sign.py.
//
//   v2_sign_encode_kernel      one CTA per PS tile (= one destination owner), one warp per bucket: bf16 gradient read
//                              in place through the pointer table with 16-byte loads where aligned; pass 1 sums |x| in
//                              fp64 in a fixed lane / butterfly order and stores scale = fp32(L1 / blen); pass 2 packs
//                              bit i of word j = (element 64 j + i < 0), each lane holding 8 elements and 8 lanes
//                              making one word; words + scales are stored into the owner's arena (the QSGD slot), then
//                              the tile's step stamp; the last CTA of the launch publishes flag[group][worker] = step on
//                              every owner.  The group's only launch.
//   v2_sign_encode_ef_kernel   the same encode plus the error-feedback epilogue e += x - (bit ? -scale : +scale).
//   v2_ps_sign_kernel          one launch per (group, owner): the push wait / --num-aggregate mask, stale-slot check
//                              and fp32 vector tiles of v2_ps_common.cuh; the counted workers' buckets are decoded and
//                              summed in fixed worker order, times 1/#counted, then the fused optimizer epilogue and
//                              the bf16 broadcast.
//   v2_sign_code_stats_kernel  --code-stats: per tile gsq = sum x^2 and mse = sum (x - decode)^2 in fp64 with the scale
//                              read back from this worker's slot (the error of the code is exact, not an expectation);
//                              atoms = numel.  The unit's last tile adds the partials in tile order.
#include "v2_bf16_load.cuh"
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int SE_THREADS = 256;
constexpr int SE_WARPS = SE_THREADS / 32;
constexpr int SPS_THREADS = 256;
constexpr int SPS_TILE_ELEMS = 4096;
constexpr int SST_MAX_BUCKETS = SPS_TILE_ELEMS / 64;

__device__ __forceinline__ float sign_decode(float x, float scale) { return x < 0.f ? -scale : scale; }

template <bool EF>
__device__ __forceinline__ void sign_encode(const PushArgs& a) {
  __shared__ float s_scale[SST_MAX_BUCKETS];
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();
  const __nv_bfloat16* gb = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off;
  const int bucket = u.K, L = u.cols;
  const int step = a.ctrl->step;
  const int jt = t.owner;                                   // encode tiles: index of the tile inside its unit
  const int owner = (u.own0 + jt) % a.n_owners;
  float* slot = a.arena_peer[owner] + (long long)a.worker * a.arena_floats + u.slot_off;
  float* scales = slot + qsgd_norms_off(u.n_ps);
  unsigned long long* words = reinterpret_cast<unsigned long long*>(slot + qsgd_words_off(u.n_ps, u.rows));
  const int kb0 = t.a / bucket, nbt = (t.b + bucket - 1) / bucket;

  // pass 1 for every bucket of the warp, then pass 2 (the fp64 division's slow path is a call: nothing of pass 2 is
  // live across it)
  for (int kb = warp; kb < nbt; kb += SE_WARPS) {
    const long long bk = kb0 + kb;
    const long long e0 = bk * bucket;
    const int blen = (int)min((long long)bucket, (long long)u.numel - e0);
    const __nv_bfloat16* src = gb + e0;
    const int nch = (((reinterpret_cast<uintptr_t>(src) & 15) | (e0 & 7)) == 0) ? (blen >> 3) : 0;
    const int nct = (blen + 7) >> 3;                        // chunks holding real elements
    // L1 in fp64, lane l over chunks l, l + 32, ... in order, then a butterfly: the same bits on every run
    double acc = 0.0;
    for (int c = lane; c < nct; c += 32) {
      float x[8];
      sign_load8(src, c, nch, blen, x);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc += (double)fabsf(x[i]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    const float scale = __double2float_rn(acc / (double)blen);
    if (lane == 0) { s_scale[kb] = scale; scales[bk] = scale; }
  }
  __syncwarp();
  for (int kb = warp; kb < nbt; kb += SE_WARPS) {
    const long long bk = kb0 + kb;
    const long long e0 = bk * bucket;
    const int blen = (int)min((long long)bucket, (long long)u.numel - e0);
    const __nv_bfloat16* src = gb + e0;
    const int nch = (((reinterpret_cast<uintptr_t>(src) & 15) | (e0 & 7)) == 0) ? (blen >> 3) : 0;
    const int nct = (blen + 7) >> 3;
    const float scale = s_scale[kb];
    float* res = EF ? a.residual + u.w_off + e0 : nullptr;
    // pass 2: lane c holds byte (c & 7) of word c >> 3; every word of the bucket is written (padding bits 0)
    for (int c0 = 0; c0 < 8 * L; c0 += 32) {
      const int c = c0 + lane;
      uint32_t byte = 0;
      if (c < nct) {
        float x[8];
        sign_load8(src, c, nch, blen, x);
#pragma unroll
        for (int i = 0; i < 8; ++i) byte |= (x[i] < 0.f ? 1u : 0u) << i;
        if (EF) {                    // e += x - g_hat; 32-byte aligned (w_off % 64 == 0, e0 % 64 == 0)
          if (c < nch) {
            float4* rp = reinterpret_cast<float4*>(res + 8 * c);
            float4 r0 = rp[0], r1 = rp[1];
            r0.x += x[0] - sign_decode(x[0], scale);
            r0.y += x[1] - sign_decode(x[1], scale);
            r0.z += x[2] - sign_decode(x[2], scale);
            r0.w += x[3] - sign_decode(x[3], scale);
            r1.x += x[4] - sign_decode(x[4], scale);
            r1.y += x[5] - sign_decode(x[5], scale);
            r1.z += x[6] - sign_decode(x[6], scale);
            r1.w += x[7] - sign_decode(x[7], scale);
            rp[0] = r0; rp[1] = r1;
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i)
              if (8 * c + i < blen) res[8 * c + i] += x[i] - sign_decode(x[i], scale);
          }
        }
      }
      unsigned long long w = (unsigned long long)byte << (8 * (lane & 7));
      w |= __shfl_xor_sync(0xffffffffu, w, 1);
      w |= __shfl_xor_sync(0xffffffffu, w, 2);
      w |= __shfl_xor_sync(0xffffffffu, w, 4);
      if ((lane & 7) == 0 && (c >> 3) < L) words[bk * L + (c >> 3)] = w;
    }
  }

  // ---- the tile's step stamp (after its words and scales), then the group's push flag -----------------------
  __syncthreads();
  if (tid == 0) {
    enc_stamp(reinterpret_cast<int*>(slot), jt, step);
    enc_push_flag(a, step);
  }
}

__global__ void __launch_bounds__(SE_THREADS) v2_sign_encode_kernel(const PushArgs a) { sign_encode<false>(a); }
// error feedback: the same encode plus the residual epilogue
__global__ void __launch_bounds__(SE_THREADS) v2_sign_encode_ef_kernel(const PushArgs a) { sign_encode<true>(a); }

// ---- PS: decode + sum + optimizer --------------------------------------------------------------------------
template <class A>
__device__ __forceinline__ void ps_sign(const A& a) {
  __shared__ __align__(16) float OUT[SPS_TILE_ELEMS];   // summed decodes of one tile, physical element order
  __shared__ int s_ok, s_bad;
  __shared__ unsigned int s_mask, s_use;
  __shared__ long long s_t_enter, s_t_ready;            // live across the whole launch: kept out of registers
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
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
    if (u.kind != KIND_SIGN) continue;
    const int bucket = u.K, L = u.cols;
    const int kb0 = t.a / bucket, nbt = (t.b + bucket - 1) / bucket;
    const int jt = kb0 / u.cs;
    const long long soff = qsgd_norms_off(u.n_ps), woff = qsgd_words_off(u.n_ps, u.rows);
    __syncthreads();   // previous tile is done with OUT / s_use
    if (tid == 0) s_use = ps_fresh_workers(a, u, jt, wmask, step, s_bad);
    for (int i = tid; i < t.b; i += blockDim.x) OUT[i] = 0.f;
    __syncthreads();
    const unsigned int use = s_use;
    // one warp per bucket; the bucket's 32-bit half words are loaded one per lane and broadcast with a shuffle, so
    // lane l owns elements l, l + 32, ... and the per-element sum over workers runs in worker order
    for (int kb = warp; kb < nbt; kb += blockDim.x >> 5) {
      const long long bk = kb0 + kb;
      const int blen = min(bucket, t.b - kb * bucket);
      float* o = OUT + kb * bucket;
      for (int w = 0; w < a.W; ++w) {
        if (!((use >> w) & 1u)) continue;
        const float* sw = a.arenas + (long long)w * a.arena_floats + u.slot_off;
        const float scale = ld_cg_f(sw + soff + bk);
        const int* hw = reinterpret_cast<const int*>(sw + woff) + 2 * bk * L;
        for (int h0 = 0; h0 < 2 * L; h0 += 32) {
          const uint32_t mine = (h0 + lane < 2 * L) ? (uint32_t)ld_cg_i(hw + h0 + lane) : 0u;
          const int nh = min(32, 2 * L - h0);
          for (int k = 0; k < nh; ++k) {
            const uint32_t v = __shfl_sync(0xffffffffu, mine, k);
            const int i = 32 * (h0 + k) + lane;
            if (i < blen) o[i] = __fadd_rn(o[i], ((v >> lane) & 1u) ? -scale : scale);
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
  if (tid == 0) ps_complete(a, ctrl, step, s_bad != 0, s_t_enter, s_t_ready);
}

__global__ void __launch_bounds__(SPS_THREADS) v2_ps_sign_kernel(const PsArgs2 a) { ps_sign(a); }
__global__ void __launch_bounds__(SPS_THREADS, 1) v2_ps_sign_lw_kernel(const PsArgsLw a) { ps_sign(a); }
__global__ void __launch_bounds__(SPS_THREADS, 1) v2_ps_sign_gather_kernel(const PsArgsGather a) { ps_sign(a); }
__global__ void __launch_bounds__(SPS_THREADS, 1) v2_ps_sign_lion_kernel(const PsArgsLion a) { ps_sign(a); }

// ---- --code-stats ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SE_THREADS) v2_sign_code_stats_kernel(const ScaleStatArgs a) {
  __shared__ double red[2][SE_WARPS];
  __shared__ float s_scale[SST_MAX_BUCKETS];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  if (u.kind != KIND_SIGN) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int jt = t.owner;
  const float* slot = a.arena_peer[(u.own0 + jt) % a.n_owners] + (long long)a.worker * a.arena_floats + u.slot_off;
  const int bucket = u.K, kb0 = t.a / bucket, nbt = (t.b + bucket - 1) / bucket;
  for (int kb = tid; kb < nbt; kb += SE_THREADS) s_scale[kb] = ld_cg_f(slot + qsgd_norms_off(u.n_ps) + kb0 + kb);
  __syncthreads();
  const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a;
  double gsq = 0.0, mse = 0.0;
  for (int i = tid; i < t.b; i += SE_THREADS) {
    const float x = sign_ftz(__bfloat162float(src[i]));
    const double xd = (double)x, d = xd - (double)sign_decode(x, s_scale[i / bucket]);
    gsq = fma(xd, xd, gsq);
    mse = fma(d, d, mse);
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
    for (int w = 0; w < SE_WARPS; ++w) { g += red[0][w]; m += red[1][w]; }
    stat_store_tile(a, u, g, m, (double)t.b, 0.0, (double)t.b, s_last);   // every element is an atom
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

extern "C" {

void atomo_v2_launch_sign_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 float* const* arena_peer, int* const* sig_peer, int n_owners, long long arena_floats,
                                 int worker, int group, const void* ctrl, unsigned int* group_counter,
                                 long long* tstats, int final_group, float* residual, cudaStream_t stream) {
  if (ntiles <= 0) return;
  PushArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.tstats = tstats; a.final_group = final_group; a.residual = residual;
  if (residual != nullptr) v2_sign_encode_ef_kernel<<<ntiles, SE_THREADS, 0, stream>>>(a);
  else v2_sign_encode_kernel<<<ntiles, SE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_sign(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                             int final_group, int owner, float* master, float* mom, float* sq, float* sqmax,
                             float* vmom, float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer,
                             float* vparams_local, float* vparams_mc, float* const* vparams_peer,
                             const float* vgrads_mc, const float* const* vgrads_peer, const float* arenas,
                             long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                             unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                             cudaStream_t stream) {
  v2_ps_sign_kernel<<<ps_grid(grid, ntiles), SPS_THREADS, 0, stream>>>(
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, final_group, owner, master, mom, sq, sqmax, vmom, vsq,
              vsqmax, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, vgrads_mc, vgrads_peer,
              nullptr, arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w));
}

void atomo_v2_launch_sign_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                     const long long* gptr, float* const* arena_peer, int n_owners,
                                     long long arena_floats, int worker, double* partials, unsigned int* unit_counters,
                                     double* acc, cudaStream_t stream) {
  if (ntiles <= 0) return;
  ScaleStatArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr;
  a.arena_peer = arena_peer; a.n_owners = n_owners; a.arena_floats = arena_floats; a.worker = worker;
  a.partials = partials; a.unit_counters = unit_counters; a.acc = acc;
  v2_sign_code_stats_kernel<<<ntiles, SE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_sign_lw(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLw& a = *static_cast<const PsArgsLw*>(args);
  v2_ps_sign_lw_kernel<<<ps_grid(grid, a.ntiles), SPS_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_sign_gather(const void* args, int grid, cudaStream_t stream) {
  const PsArgsGather& a = *static_cast<const PsArgsGather*>(args);
  v2_ps_sign_gather_kernel<<<ps_grid(grid, a.ntiles), SPS_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_sign_lion(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLion& a = *static_cast<const PsArgsLion*>(args);
  v2_ps_sign_lion_kernel<<<ps_grid(grid, a.ntiles), SPS_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
