// FP8 (e4m3) with stochastic rounding on the overlapped, sharded bf16 engine (sm_90a): worker-side encode + push of
// ONE backward group, the owner-side decode + optimizer step, and --code-stats.  The oracle is codings/fp8.py.
//
//   v2_fp8_encode_kernel      one CTA per PS tile (= one destination owner); each thread takes groups of 16 elements
//                             (two 16-byte bf16 loads where aligned).  Pass 1: the largest magnitude of every bucket as
//                             an integer max of the magnitude bits in shared memory (Inf / NaN bits are the largest,
//                             so the special test needs no fmaxf); the scale 2^-k of each bucket.  Pass 2: y = |x| 2^k,
//                             its e4m3 neighbours lo / hi and one Philox uniform per element (keyed by seed / element /
//                             unit / step / worker) choose hi with probability (y - lo) / ulp; the signed values go to
//                             bytes with the hardware conversion (cvt.rn.satfinite.e4m3x2.f32, exact here), one 16-byte
//                             store per group.  Bytes + scales land in the owner's arena (the QSGD slot), then the
//                             tile's step stamp; the last CTA of the launch publishes flag[group][worker] = step on
//                             every owner.  The group's only launch.
//   v2_fp8_encode_ef_kernel   the same encode plus the error-feedback epilogue e += x - decode(byte) * scale, from the
//                             byte and scale pushed.
//   v2_ps_fp8_kernel          one launch per (group, owner): the push wait / --num-aggregate mask, stale-slot check
//                             and fp32 vector tiles of v2_ps_common.cuh; each thread decodes 16 elements of every
//                             counted worker (cvt.rn.f16x2.e4m3x2, then an exact fp32 product with the scale), sums
//                             them in fixed worker order, times 1/#counted, and runs the fused optimizer epilogue and
//                             the bf16 broadcast from registers.
//   v2_fp8_code_stats_kernel  --code-stats: per tile gsq = sum x^2 and the expected error sum (y - lo)(hi - y) 2^-2k
//                             in fp64, with the scale read back from this worker's slot; atoms = numel.  The unit's
//                             last tile adds the partials in tile order.
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "v2_bf16_load.cuh"
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int FE_THREADS = 256;
constexpr int FE_WARPS = FE_THREADS / 32;
constexpr int FPS_THREADS = 256;
constexpr int F_TILE_ELEMS = 4096;
constexpr int F_MAX_BUCKETS = F_TILE_ELEMS / 64;
constexpr unsigned long long FP8_KEY_XOR = 0xF8E43A5C96D1B207ULL;   // codings/fp8.py FP8_KEY_XOR
constexpr uint32_t FP8_SPECIAL_BITS = 0x7e800000u;   // 2^126: a bucket max at or above it (Inf, NaN) -> scale NaN
constexpr int FP8_K_MAX = 117;                       // 2^-9 * 2^-117 = 2^-126: decoded values stay fp32 normals

// scale 2^-k of a bucket from the bits of its largest magnitude: amax 2^k in (224, 448], k <= 117; 0 for an all-zero
// bucket, NaN for a bucket holding an Inf or NaN or with amax >= 2^126
__device__ __forceinline__ float fp8_scale(uint32_t ab) {
  if (ab == 0u) return 0.f;
  if (ab >= FP8_SPECIAL_BITS) return __uint_as_float(0x7fc00000u);
  const int e = (int)(ab >> 23) - 127;
  const int k = min(((ab & 0x7fffffu) > 0x600000u ? 7 : 8) - e, FP8_K_MAX);
  return __uint_as_float((uint32_t)(127 - k) << 23);
}

// 2^k of a finite, non-zero scale 2^-k (exact)
__device__ __forceinline__ float fp8_inv_pow2(float s) { return __uint_as_float((254u << 23) - __float_as_uint(s)); }

// y = |x| 2^k (exact; below 2^-126 it counts as zero), its lower e4m3 neighbour lo, the spacing ulp above lo and
// p = (y - lo) / ulp, every step exact
__device__ __forceinline__ void fp8_neighbours(float ax, float pk, float& y, float& lo, float& ulp, float& p) {
  y = ax * pk;
  if (!(y >= 0x1p-126f)) y = 0.f;
  if (y >= 0x1p-6f) {
    const uint32_t yb = __float_as_uint(y);
    lo = __uint_as_float(yb & 0xfff00000u);                      // mantissa truncated to 3 bits
    ulp = __uint_as_float((yb & 0x7f800000u) - (3u << 23));
    p = (y - lo) * fp8_inv_pow2(ulp);
  } else {
    const float t = y * 512.f;
    const float f = floorf(t);
    lo = f * 0x1p-9f;
    ulp = 0x1p-9f;
    p = t - f;
  }
}

// the signed value pushed for x: hi = lo + ulp when u < p, else lo; a zero result is +0 (byte 0x00)
__device__ __forceinline__ float fp8_round(float x, float pk, float u) {
  float y, lo, ulp, p;
  fp8_neighbours(fabsf(x), pk, y, lo, ulp, p);
  const float v = u < p ? lo + ulp : lo;
  return (x < 0.f && v > 0.f) ? -v : v;
}

// two exactly representable values to two e4m3 bytes (a in the low byte)
__device__ __forceinline__ uint32_t fp8_pack2(float a, float b) {
  return (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
}

// four e4m3 bytes (byte 0 first) to fp32, exactly
__device__ __forceinline__ void fp8_unpack4(uint32_t w, float* f) {
  const __half2_raw lo = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w & 0xffffu), __NV_E4M3);
  const __half2_raw hi = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w >> 16), __NV_E4M3);
  const float2 a = __half22float2(__half2(lo)), b = __half22float2(__half2(hi));
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
}

template <bool EF>
__device__ __forceinline__ void fp8_encode(const PushArgs& a) {
  __shared__ unsigned int s_amax[F_MAX_BUCKETS];
  __shared__ float s_scale[F_MAX_BUCKETS];
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();
  const int bucket = u.K, L = u.cols;
  const int step = a.ctrl->step;
  const int jt = t.owner;                                   // encode tiles: index of the tile inside its unit
  const int owner = (u.own0 + jt) % a.n_owners;
  float* slot = a.arena_peer[owner] + (long long)a.worker * a.arena_floats + u.slot_off;
  float* scales = slot + qsgd_norms_off(u.n_ps);
  const int kb0 = t.a / bucket, nbt = (t.b + bucket - 1) / bucket;
  // element i of the tile is byte kb0 * 8L + i (bucket == 8L, or the tensor is one bucket); 16-byte aligned
  unsigned char* bytes = reinterpret_cast<unsigned char*>(slot + qsgd_words_off(u.n_ps, u.rows)) + (long long)kb0 * 8 * L;
  const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a;
  const int nch = (reinterpret_cast<uintptr_t>(src) & 15) == 0 ? (t.b >> 3) : 0;   // t.a % 64 == 0
  const int nbytes = nbt * 8 * L;                          // every byte of the tile's buckets, padding included
  const int ng = (nbytes + 15) >> 4;

  for (int kb = tid; kb < nbt; kb += FE_THREADS) s_amax[kb] = 0u;
  __syncthreads();
  // pass 1: the largest magnitude of each bucket (a group of 16 lies in one bucket: bucket % 64 == 0 or one bucket)
  for (int gi = tid; 16 * gi < t.b; gi += FE_THREADS) {
    float x[2][8];
    sign_load8(src, 2 * gi, nch, t.b, x[0]);
    sign_load8(src, 2 * gi + 1, nch, t.b, x[1]);
    uint32_t m = 0u;
#pragma unroll
    for (int i = 0; i < 16; ++i) m = max(m, __float_as_uint(x[i >> 3][i & 7]) & 0x7fffffffu);
    atomicMax(&s_amax[16 * gi / bucket], m);
  }
  __syncthreads();
  for (int kb = tid; kb < nbt; kb += FE_THREADS) {
    const float s = fp8_scale(s_amax[kb]);
    s_scale[kb] = s;
    scales[kb0 + kb] = s;
  }
  __syncthreads();
  // pass 2: round, pack, store (and the residual)
  float* res = EF ? a.residual + u.w_off + t.a : nullptr;
  const unsigned long long key = a.ctrl->seed ^ FP8_KEY_XOR;
  for (int gi = tid; gi < ng; gi += FE_THREADS) {
    const int i0 = 16 * gi;
    float x[2][8];
    sign_load8(src, 2 * gi, nch, t.b, x[0]);
    sign_load8(src, 2 * gi + 1, nch, t.b, x[1]);
    const int kb = min(i0 / bucket, nbt - 1);
    const float scale = s_scale[kb];
    uint32_t w[4] = {0u, 0u, 0u, 0u};
    if (scale > 0.f) {                                     // 0: all zero, NaN: special -> zero bytes
      const float pk = fp8_inv_pow2(scale);
      const long long e0 = (long long)t.a + i0;            // element index in the unit; e0 % 16 == 0
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        uint32_t r4[4];
        Philox::gen(key, (uint32_t)((e0 >> 2) + q), (uint32_t)t.unit, (uint32_t)step, (uint32_t)a.worker, r4);
        const float* xq = &x[q >> 1][4 * (q & 1)];
        const float v0 = fp8_round(xq[0], pk, Philox::to_uniform(r4[0]));
        const float v1 = fp8_round(xq[1], pk, Philox::to_uniform(r4[1]));
        const float v2 = fp8_round(xq[2], pk, Philox::to_uniform(r4[2]));
        const float v3 = fp8_round(xq[3], pk, Philox::to_uniform(r4[3]));
        w[q] = fp8_pack2(v0, v1) | (fp8_pack2(v2, v3) << 16);
      }
    }
    if (i0 + 16 <= nbytes) *reinterpret_cast<uint4*>(bytes + i0) = make_uint4(w[0], w[1], w[2], w[3]);
    else *reinterpret_cast<uint2*>(bytes + i0) = make_uint2(w[0], w[1]);   // nbytes % 8 == 0
    if (EF && i0 < t.b) {            // e += x - decode(byte) * scale; 64-byte aligned (w_off % 64 == 0, t.a % 64 == 0)
      float d[16];
#pragma unroll
      for (int q = 0; q < 4; ++q) fp8_unpack4(w[q], d + 4 * q);
#pragma unroll
      for (int i = 0; i < 16; ++i) d[i] = x[i >> 3][i & 7] - __fmul_rn(d[i], scale);
      if (i0 + 16 <= t.b) {
        float4* rp = reinterpret_cast<float4*>(res + i0);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float4 r = rp[q];
          r.x += d[4 * q]; r.y += d[4 * q + 1]; r.z += d[4 * q + 2]; r.w += d[4 * q + 3];
          rp[q] = r;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i)
          if (i0 + i < t.b) res[i0 + i] += d[i];
      }
    }
  }

  // ---- the tile's step stamp (after its bytes and scales), then the group's push flag -----------------------
  __syncthreads();
  if (tid == 0) {
    enc_stamp(reinterpret_cast<int*>(slot), jt, step);
    enc_push_flag(a, step);
  }
}

__global__ void __launch_bounds__(FE_THREADS) v2_fp8_encode_kernel(const PushArgs a) { fp8_encode<false>(a); }
// error feedback: the same encode plus the residual epilogue
__global__ void __launch_bounds__(FE_THREADS) v2_fp8_encode_ef_kernel(const PushArgs a) { fp8_encode<true>(a); }

// ---- PS: decode + sum + optimizer --------------------------------------------------------------------------
template <class A>
__device__ __forceinline__ void ps_fp8(const A& a) {
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
    if (u.kind != KIND_FP8) continue;
    const int bucket = u.K, L = u.cols;
    const int kb0 = t.a / bucket;
    const int jt = kb0 / u.cs;
    const long long soff = qsgd_norms_off(u.n_ps) + kb0;
    const long long boff = 4LL * qsgd_words_off(u.n_ps, u.rows) + (long long)kb0 * 8 * L;   // bytes
    __syncthreads();   // previous tile is done with s_use
    if (tid == 0) s_use = ps_fresh_workers(a, u, jt, wmask, step, s_bad);
    __syncthreads();
    const unsigned int use = s_use;
    const long long e0 = u.w_off + t.a;                  // % 64 == 0
    // 16 elements per thread and step: one 16-byte load of bytes per counted worker, all in one bucket
    for (int i0 = 16 * tid; i0 < t.b; i0 += 16 * blockDim.x) {
      const int kb = i0 / bucket;
      float g[2][8];
#pragma unroll
      for (int i = 0; i < 16; ++i) g[i >> 3][i & 7] = 0.f;
      for (int w = 0; w < a.W; ++w) {
        if (!((use >> w) & 1u)) continue;
        const float* sw = a.arenas + (long long)w * a.arena_floats + u.slot_off;
        const float scale = ld_cg_f(sw + soff + kb);
        const uint4 q = ld_cg_u4(reinterpret_cast<const unsigned char*>(sw) + boff + i0);
        const uint32_t qw[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          float d[4];
          fp8_unpack4(qw[h], d);
#pragma unroll
          for (int i = 0; i < 4; ++i) g[h >> 1][4 * (h & 1) + i] = __fadd_rn(g[h >> 1][4 * (h & 1) + i], __fmul_rn(d[i], scale));
        }
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) g[i >> 3][i & 7] *= inv_w;
      if (i0 + 16 <= t.b) {
        update8(a, c, e0 + i0, g[0]);
        update8(a, c, e0 + i0 + 8, g[1]);
      } else {
        for (int i = 0; i < 16 && i0 + i < t.b; ++i) update1(a, c, e0 + i0 + i, g[i >> 3][i & 7]);
      }
    }
    lw_tile_done(a, ti);
  }

  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, s_bad != 0, s_t_enter, s_t_ready);
}

__global__ void __launch_bounds__(FPS_THREADS) v2_ps_fp8_kernel(const PsArgs2 a) { ps_fp8(a); }
__global__ void __launch_bounds__(FPS_THREADS, 1) v2_ps_fp8_lw_kernel(const PsArgsLw a) { ps_fp8(a); }
__global__ void __launch_bounds__(FPS_THREADS, 1) v2_ps_fp8_gather_kernel(const PsArgsGather a) { ps_fp8(a); }
__global__ void __launch_bounds__(FPS_THREADS, 1) v2_ps_fp8_lion_kernel(const PsArgsLion a) { ps_fp8(a); }

// ---- --code-stats ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FE_THREADS) v2_fp8_code_stats_kernel(const ScaleStatArgs a) {
  __shared__ double red[2][FE_WARPS];
  __shared__ float s_scale[F_MAX_BUCKETS];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  if (u.kind != KIND_FP8) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int jt = t.owner;
  const float* slot = a.arena_peer[(u.own0 + jt) % a.n_owners] + (long long)a.worker * a.arena_floats + u.slot_off;
  const int bucket = u.K, kb0 = t.a / bucket, nbt = (t.b + bucket - 1) / bucket;
  for (int kb = tid; kb < nbt; kb += FE_THREADS) s_scale[kb] = ld_cg_f(slot + qsgd_norms_off(u.n_ps) + kb0 + kb);
  __syncthreads();
  const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a;
  double gsq = 0.0, mse = 0.0;
  for (int i = tid; i < t.b; i += FE_THREADS) {
    const float x = sign_ftz(__bfloat162float(src[i]));
    const float s = s_scale[i / bucket];
    const double xd = (double)x;
    gsq = fma(xd, xd, gsq);
    if (!(s > 0.f)) {                                     // zero bucket: no error; special bucket: NaN
      if (s != 0.f) mse += (double)s;
      continue;
    }
    float y, lo, ulp, p;
    fp8_neighbours(fabsf(x), fp8_inv_pow2(s), y, lo, ulp, p);
    const double sd = (double)s;
    mse = fma((double)(y - lo) * (double)(lo + ulp - y), sd * sd, mse);
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
    for (int w = 0; w < FE_WARPS; ++w) { g += red[0][w]; m += red[1][w]; }
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

void atomo_v2_launch_fp8_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                float* const* arena_peer, int* const* sig_peer, int n_owners, long long arena_floats,
                                int worker, int group, const void* ctrl, unsigned int* group_counter,
                                long long* tstats, int final_group, float* residual, cudaStream_t stream) {
  if (ntiles <= 0) return;
  PushArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.tstats = tstats; a.final_group = final_group; a.residual = residual;
  if (residual != nullptr) v2_fp8_encode_ef_kernel<<<ntiles, FE_THREADS, 0, stream>>>(a);
  else v2_fp8_encode_kernel<<<ntiles, FE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_fp8(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                            int final_group, int owner, float* master, float* mom, float* sq, float* sqmax,
                            float* vmom, float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer,
                            float* vparams_local, float* vparams_mc, float* const* vparams_peer,
                            const float* vgrads_mc, const float* const* vgrads_peer, const float* arenas,
                            long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                            unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                            cudaStream_t stream) {
  v2_ps_fp8_kernel<<<ps_grid(grid, ntiles), FPS_THREADS, 0, stream>>>(
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, final_group, owner, master, mom, sq, sqmax, vmom, vsq,
              vsqmax, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, vgrads_mc, vgrads_peer,
              nullptr, arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w));
}

void atomo_v2_launch_fp8_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                    const long long* gptr, float* const* arena_peer, int n_owners,
                                    long long arena_floats, int worker, double* partials, unsigned int* unit_counters,
                                    double* acc, cudaStream_t stream) {
  if (ntiles <= 0) return;
  ScaleStatArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr;
  a.arena_peer = arena_peer; a.n_owners = n_owners; a.arena_floats = arena_floats; a.worker = worker;
  a.partials = partials; a.unit_counters = unit_counters; a.acc = acc;
  v2_fp8_code_stats_kernel<<<ntiles, FE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_fp8_lw(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLw& a = *static_cast<const PsArgsLw*>(args);
  v2_ps_fp8_lw_kernel<<<ps_grid(grid, a.ntiles), FPS_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_fp8_gather(const void* args, int grid, cudaStream_t stream) {
  const PsArgsGather& a = *static_cast<const PsArgsGather*>(args);
  v2_ps_fp8_gather_kernel<<<ps_grid(grid, a.ntiles), FPS_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_fp8_lion(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLion& a = *static_cast<const PsArgsLion*>(args);
  v2_ps_fp8_lion_kernel<<<ps_grid(grid, a.ntiles), FPS_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
