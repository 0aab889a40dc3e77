// Randomized-Hadamard rotated quantization on the overlapped, sharded bf16 engine (sm_90a): worker-side encode + push
// of ONE backward group, the owner-side decode + inverse rotation + optimizer step, and --code-stats.  The oracle is
// codings/hadamard.py; every fp32 rounding below is a named intrinsic (the extension builds with --use_fast_math, so
// plain operators could be contracted or approximated) and the oracle mirrors each one, flush-to-zero included.
//
// Every kernel runs 256 threads on one PS tile of at most 4096 elements (max(1, 4096 / d) whole buckets of d = 64 ..
// 4096 elements); thread i holds elements 16 i .. 16 i + 15 of the tile in registers.  The butterflies of H_d run in
// the oracle's stage order h = 1, 2, ..., d / 2: h < 16 inside a thread, 16 <= h <= 256 across lanes with
// __shfl_xor_sync, h >= 512 across warps through a transpose in shared memory.
//
//   v2_hadamard_encode_kernel      one CTA per PS tile (= one destination owner): 16-byte bf16 loads, the Philox
//                                  signs (keyed by seed / element / unit / step, no worker: every worker rotates a
//                                  bucket the same way), the forward butterflies, min / max per bucket (a non-finite
//                                  bucket stores lo = step = NaN), stochastic rounding to 2^bits levels with one Philox
//                                  uniform per element (keyed by seed / element / unit / step / worker), codes packed
//                                  in element order and stored with one 4 / 8 / 16-byte store per thread; (lo, step)
//                                  and the codes land in the owner's arena, then the tile's step stamp; the last CTA of
//                                  the launch publishes flag[group][worker] = step on every owner.  The group's only
//                                  launch.
//   v2_hadamard_encode_ef_kernel   the same encode plus the error-feedback epilogue e += x - s H y_hat / d over the real
//                                  elements: one inverse transform of this worker's own decode.
//   v2_ps_hadamard_kernel          one launch per (group, owner): the push wait / --num-aggregate mask, stale-slot
//                                  check and fp32 vector tiles of v2_ps_common.cuh; each thread decodes y_hat =
//                                  fma(c, step, lo) of every counted worker and sums them in fixed worker order in the
//                                  rotated domain, then one inverse transform per bucket, * 2^-log2(d), * s, * 1 /
//                                  #counted, and the fused optimizer epilogue and bf16 broadcast from registers.
//   v2_hadamard_code_stats_kernel  --code-stats: per tile gsq = sum x^2 and the expected error
//                                  sum_b (n_b / d^2) sum_i f_i (1 - f_i) step_b^2 in fp64, recomputing the rotation and
//                                  reading (lo, step) back from this worker's slot; atoms = numel.  The unit's last
//                                  tile adds the partials in tile order.
#include "v2_bf16_load.cuh"
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int HD_THREADS = 256;
constexpr int HD_WARPS = HD_THREADS / 32;
constexpr int HD_TILE = 16 * HD_THREADS;                              // 4096 elements: the largest tile
constexpr unsigned long long HD_ROT_KEY = 0x48D2A7E13B5C9F61ULL;     // codings/hadamard.py HADAMARD_ROT_KEY
constexpr unsigned long long HD_Q_KEY = 0x7C1E94B2D58A3F0DULL;       // codings/hadamard.py HADAMARD_Q_KEY
constexpr float HD_FLT_MIN = 0x1p-126f;

// float offsets inside a hadamard slot (ops/plan2.py hadamard_params_off / hadamard_words_off)
__device__ __forceinline__ long long hd_params_off(int n_ps) { return (n_ps + 3) & ~3; }
__device__ __forceinline__ long long hd_words_off(int n_ps, int buckets) {
  return hd_params_off(n_ps) + ((2LL * buckets + 3) & ~3LL);
}

struct HdShared {
  float x[HD_TILE];                          // the cross-warp butterfly stages
  float wlo[HD_WARPS], whi[HD_WARPS];        // per-warp min / max of buckets wider than a warp
  int wbad[HD_WARPS];
};

struct HdRange {
  float lo, step;
};

// a zero of either sign read as +0 (by bits: the comparison would not tell them apart)
__device__ __forceinline__ float hd_pos0(float x) { return (__float_as_uint(x) & 0x7fffffffu) ? x : 0.f; }
__device__ __forceinline__ bool hd_nonfinite(float x) { return (__float_as_uint(x) & 0x7f800000u) == 0x7f800000u; }

// the 16 rotation signs of elements e0 .. e0 + 15 (e0 % 16 == 0): bit e & 31 of word (e >> 5) & 3 of
// Philox(seed ^ HD_ROT_KEY, (e >> 7, unit, step, 0)); bit r of the result negates element e0 + r
__device__ __forceinline__ uint32_t hd_signs(unsigned long long seed, long long e0, int unit, int step) {
  uint32_t r4[4];
  Philox::gen(seed ^ HD_ROT_KEY, (uint32_t)(e0 >> 7), (uint32_t)unit, (uint32_t)step, 0u, r4);
  const int q = (int)(e0 >> 5) & 3;
  const uint32_t w = q == 0 ? r4[0] : q == 1 ? r4[1] : q == 2 ? r4[2] : r4[3];
  return (w >> (uint32_t)(e0 & 31)) & 0xffffu;
}

// H_d on every bucket of the tile, in place: stages h = 1 .. d / 2 of (a, b) -> (a + b, a - b).  Every thread of the
// CTA calls it (shuffles and barriers).
__device__ __forceinline__ void hd_butterflies(float (&v)[16], int d, float* sx) {
  const int tid = threadIdx.x, lane = tid & 31;
#pragma unroll
  for (int h = 1; h < 16; h <<= 1) {
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      if (r & h) continue;
      const float a = v[r], b = v[r + h];
      v[r] = __fadd_rn(a, b);
      v[r + h] = __fsub_rn(a, b);
    }
  }
#pragma unroll
  for (int m = 1; m < 32; m <<= 1) {            // h = 16 m: the partner is lane ^ m
    if (16 * m >= d) break;
    const bool up = (lane & m) != 0;
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const float p = __shfl_xor_sync(0xffffffffu, v[r], m);
      v[r] = up ? __fsub_rn(p, v[r]) : __fadd_rn(v[r], p);
    }
  }
  if (d > 512) {                                 // h = 512 .. d / 2: thread j takes elements j + 256 k, k = 0 .. 15
    float4* s4 = reinterpret_cast<float4*>(sx) + 4 * tid;
#pragma unroll
    for (int q = 0; q < 4; ++q) s4[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    __syncthreads();
    float w[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) w[k] = sx[tid + HD_THREADS * k];
#pragma unroll
    for (int m = 2; m < 16; m <<= 1) {           // h = 256 m
      if (HD_THREADS * m >= d) break;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        if (k & m) continue;
        const float a = w[k], b = w[k + m];
        w[k] = __fadd_rn(a, b);
        w[k + m] = __fsub_rn(a, b);
      }
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) sx[tid + HD_THREADS * k] = w[k];
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 f = s4[q];
      v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
    }
    __syncthreads();                             // sx is free again
  }
}

// The rotated tile of this thread: elements t.a + 16 tid .. + 15 of the unit (0 past t.b), flushed, -0 read as +0,
// signed and transformed; zeros of the result read as +0.  Returns the sign bits; x receives the flushed input.
__device__ __forceinline__ uint32_t hd_rotate(const __nv_bfloat16* src, int nch, int blen, long long e0,
                                              unsigned long long seed, int unit, int step, int d, float* sx,
                                              float (&x)[16], float (&v)[16]) {
  const int tid = threadIdx.x;
  float a[8], b[8];
  sign_load8(src, 2 * tid, nch, blen, a);
  sign_load8(src, 2 * tid + 1, nch, blen, b);
#pragma unroll
  for (int r = 0; r < 8; ++r) { x[r] = hd_pos0(a[r]); x[8 + r] = hd_pos0(b[r]); }
  const uint32_t neg = hd_signs(seed, e0, unit, step);
#pragma unroll
  for (int r = 0; r < 16; ++r) v[r] = ((neg >> r) & 1u) ? -x[r] : x[r];
  hd_butterflies(v, d, sx);
#pragma unroll
  for (int r = 0; r < 16; ++r) v[r] = hd_pos0(v[r]);
  return neg;
}

// (lo, step) of this thread's bucket: min / max over the bucket (d / 16 threads), NaN for a non-finite bucket,
// step = (hi - lo) / (L - 1) with the underflow rule (below 2^-126 it is 0).  Every thread of the CTA calls it.
__device__ __forceinline__ HdRange hd_range(const float (&v)[16], int d, int levels, HdShared& sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float mn = v[0], mx = v[0];
  int bad = 0;
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    bad |= hd_nonfinite(v[r]) ? 1 : 0;
    mn = fminf(mn, v[r]);
    mx = fmaxf(mx, v[r]);
  }
#pragma unroll
  for (int m = 1; m < 32; m <<= 1) {
    if (16 * m >= d) break;
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, m));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
    bad |= __shfl_xor_sync(0xffffffffu, bad, m);
  }
  if (d > 512) {                                 // the bucket spans d / 512 warps
    if (lane == 0) { sm.wlo[warp] = mn; sm.whi[warp] = mx; sm.wbad[warp] = bad; }
    __syncthreads();
    const int nw = d >> 9, w0 = warp / nw * nw;
    for (int w = w0; w < w0 + nw; ++w) {
      mn = fminf(mn, sm.wlo[w]);
      mx = fmaxf(mx, sm.whi[w]);
      bad |= sm.wbad[w];
    }
  }
  HdRange out;
  const float rng = __fsub_rn(mx, mn);
  if (bad || hd_nonfinite(rng)) {
    out.lo = out.step = __uint_as_float(0x7fc00000u);
  } else {
    float st = __fdiv_rn(rng, (float)(levels - 1));
    if (!(st >= HD_FLT_MIN)) st = 0.f;
    out.lo = mn;
    out.step = st;
  }
  return out;
}

// t = (y - lo) / step, each result flushed (step > 0)
__device__ __forceinline__ float hd_t(float y, float lo, float st) {
  float df = __fsub_rn(y, lo);
  if (df < HD_FLT_MIN) df = 0.f;
  float t = __fdiv_rn(df, st);
  if (t < HD_FLT_MIN) t = 0.f;
  return t;
}

template <int B>
__device__ __forceinline__ void hd_pack(const int (&c)[16], uint32_t (&pk)[4]) {
#pragma unroll
  for (int r = 0; r < 16; ++r) pk[(r * B) >> 5] |= (uint32_t)c[r] << ((r * B) & 31);
}
template <int B>
__device__ __forceinline__ void hd_unpack(const uint32_t (&pk)[4], int (&c)[16]) {
#pragma unroll
  for (int r = 0; r < 16; ++r) c[r] = (int)((pk[(r * B) >> 5] >> ((r * B) & 31)) & ((1u << B) - 1u));
}

__device__ __forceinline__ uint2 hd_ld_cg_u2(const void* p) {
  uint2 v;
  asm volatile("ld.global.cg.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}

// the 16 codes of one thread: 2 bits -> 4 bytes, 4 bits -> 8 bytes, 8 bits -> 16 bytes (aligned to their size)
__device__ __forceinline__ void hd_store_codes(unsigned char* p, int bits, const int (&c)[16]) {
  uint32_t pk[4] = {0u, 0u, 0u, 0u};
  if (bits == 2) {
    hd_pack<2>(c, pk);
    *reinterpret_cast<uint32_t*>(p) = pk[0];
  } else if (bits == 4) {
    hd_pack<4>(c, pk);
    *reinterpret_cast<uint2*>(p) = make_uint2(pk[0], pk[1]);
  } else {
    hd_pack<8>(c, pk);
    *reinterpret_cast<uint4*>(p) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
  }
}
__device__ __forceinline__ void hd_load_codes(const unsigned char* p, int bits, int (&c)[16]) {
  uint32_t pk[4] = {0u, 0u, 0u, 0u};
  if (bits == 2) {
    pk[0] = (uint32_t)ld_cg_i(reinterpret_cast<const int*>(p));
    hd_unpack<2>(pk, c);
  } else if (bits == 4) {
    const uint2 q = hd_ld_cg_u2(p);
    pk[0] = q.x; pk[1] = q.y;
    hd_unpack<4>(pk, c);
  } else {
    const uint4 q = ld_cg_u4(p);
    pk[0] = q.x; pk[1] = q.y; pk[2] = q.z; pk[3] = q.w;
    hd_unpack<8>(pk, c);
  }
}

// 2^-log2(d), exact
__device__ __forceinline__ float hd_inv_d(int d) { return __uint_as_float((uint32_t)(127 - (31 - __clz(d))) << 23); }

template <bool EF>
__device__ __forceinline__ void hadamard_encode(const PushArgs& a) {
  __shared__ __align__(16) HdShared sm;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();
  const int d = u.K, bits = u.I, levels = 1 << bits;
  const int step = a.ctrl->step;
  const unsigned long long seed = a.ctrl->seed;
  const int jt = t.owner;                                   // encode tiles: index of the tile inside its unit
  const int owner = (u.own0 + jt) % a.n_owners;
  float* slot = a.arena_peer[owner] + (long long)a.worker * a.arena_floats + u.slot_off;
  const int kb0 = t.a / d, nbt = (t.b + d - 1) / d;
  const int i0 = 16 * tid, kb = i0 / d;
  const bool live = kb < nbt;                               // a thread of a real (possibly zero-padded) bucket
  const long long e0 = (long long)t.a + i0;                 // element index in the unit
  const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a;
  const int nch = (reinterpret_cast<uintptr_t>(src) & 15) == 0 ? (t.b >> 3) : 0;   // t.a % 64 == 0

  float x[16], v[16];
  const uint32_t neg = hd_rotate(src, nch, t.b, e0, seed, t.unit, step, d, sm.x, x, v);
  const HdRange rg = hd_range(v, d, levels, sm);
  int c[16];
  {
    const unsigned long long key = seed ^ HD_Q_KEY;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint32_t r4[4];
      Philox::gen(key, (uint32_t)((e0 >> 2) + q), (uint32_t)t.unit, (uint32_t)step, (uint32_t)a.worker, r4);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = 4 * q + i;
        int cr = 0;
        if (rg.step > 0.f) {                                // 0: hi == lo or underflow; NaN: special -> code 0
          const float tt = hd_t(v[r], rg.lo, rg.step);
          const float fl = floorf(tt);
          cr = (int)fl + (Philox::to_uniform(r4[i]) < __fsub_rn(tt, fl) ? 1 : 0);
          cr = min(max(cr, 0), levels - 1);
        }
        c[r] = cr;
      }
    }
  }
  if (live) {
    if ((i0 & (d - 1)) == 0)
      *reinterpret_cast<float2*>(slot + hd_params_off(u.n_ps) + 2LL * (kb0 + kb)) = make_float2(rg.lo, rg.step);
    unsigned char* words = reinterpret_cast<unsigned char*>(slot + hd_words_off(u.n_ps, u.rows));
    hd_store_codes(words + e0 * bits / 8, bits, c);
  }
  if (EF) {                      // e += x - s H y_hat / d over the real elements
#pragma unroll
    for (int r = 0; r < 16; ++r) v[r] = __fmaf_rn((float)c[r], rg.step, rg.lo);
    hd_butterflies(v, d, sm.x);
    const float inv_d = hd_inv_d(d);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const float xh = __fmul_rn(v[r], inv_d);
      v[r] = __fsub_rn(x[r], ((neg >> r) & 1u) ? -xh : xh);
    }
    float* res = a.residual + u.w_off + t.a + i0;           // 64-byte aligned (w_off % 64 == 0, t.a % 64 == 0)
    if (i0 + 16 <= t.b) {
      float4* rp = reinterpret_cast<float4*>(res);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float4 r = rp[q];
        r.x += v[4 * q]; r.y += v[4 * q + 1]; r.z += v[4 * q + 2]; r.w += v[4 * q + 3];
        rp[q] = r;
      }
    } else {
#pragma unroll
      for (int r = 0; r < 16; ++r)
        if (i0 + r < t.b) res[r] += v[r];
    }
  }

  // ---- the tile's step stamp (after its codes and ranges), then the group's push flag ------------------------
  __syncthreads();
  if (tid == 0) {
    enc_stamp(reinterpret_cast<int*>(slot), jt, step);
    enc_push_flag(a, step);
  }
}

__global__ void __launch_bounds__(HD_THREADS) v2_hadamard_encode_kernel(const PushArgs a) { hadamard_encode<false>(a); }
// error feedback: the same encode plus the residual epilogue
__global__ void __launch_bounds__(HD_THREADS, 1) v2_hadamard_encode_ef_kernel(const PushArgs a) {
  hadamard_encode<true>(a);
}

// ---- PS: decode + sum in the rotated domain + one inverse transform + optimizer --------------------------------
template <class A>
__device__ __forceinline__ void ps_hadamard(const A& a) {
  __shared__ __align__(16) float s_x[HD_TILE];
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
  const unsigned long long seed = ctrl->seed;
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
    if (u.kind != KIND_HADAMARD) continue;
    const int d = u.K, bits = u.I;
    const int kb0 = t.a / d, nbt = (t.b + d - 1) / d;
    const int jt = kb0 / u.cs;
    const int i0 = 16 * tid, kb = i0 / d;
    const bool live = kb < nbt;
    const long long e0 = (long long)t.a + i0;
    const long long poff = hd_params_off(u.n_ps) + 2LL * (kb0 + kb);
    const long long boff = 4LL * hd_words_off(u.n_ps, u.rows) + e0 * bits / 8;   // bytes
    __syncthreads();   // previous tile is done with s_use
    if (tid == 0) s_use = ps_fresh_workers(a, u, jt, wmask, step, s_bad);
    __syncthreads();
    const unsigned int use = s_use;
    float g[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) g[r] = 0.f;
    if (live) {
      for (int w = 0; w < a.W; ++w) {
        if (!((use >> w) & 1u)) continue;
        const float* sw = a.arenas + (long long)w * a.arena_floats + u.slot_off;
        const float lo = ld_cg_f(sw + poff), st = ld_cg_f(sw + poff + 1);
        int cw[16];
        hd_load_codes(reinterpret_cast<const unsigned char*>(sw) + boff, bits, cw);
#pragma unroll
        for (int r = 0; r < 16; ++r) g[r] = __fadd_rn(g[r], __fmaf_rn((float)cw[r], st, lo));
      }
    }
    hd_butterflies(g, d, s_x);
    const float inv_d = hd_inv_d(d);
    const uint32_t neg = hd_signs(seed, e0, t.unit, step);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const float xr = __fmul_rn(g[r], inv_d);
      g[r] = __fmul_rn(((neg >> r) & 1u) ? -xr : xr, inv_w);
    }
    if constexpr (ps_tile_partials<A>) {   // the epilogue below, then the reduction every thread of the CTA reaches
      if (live && i0 < t.b) {
        const long long ew = u.w_off + e0;
        if (i0 + 16 <= t.b) {
          update8(a, c, ew, *reinterpret_cast<const float(*)[8]>(g));
          update8(a, c, ew + 8, *reinterpret_cast<const float(*)[8]>(g + 8));
        } else {
          for (int r = 0; r < 16; ++r)
            if (i0 + r < t.b) update1(a, c, ew + r, g[r]);
        }
      }
      lw_tile_done(a, ti);
      continue;
    }
    if (!live || i0 >= t.b) continue;
    const long long ew = u.w_off + e0;                   // % 16 == 0
    if (i0 + 16 <= t.b) {
      update8(a, c, ew, *reinterpret_cast<const float(*)[8]>(g));
      update8(a, c, ew + 8, *reinterpret_cast<const float(*)[8]>(g + 8));
    } else {
#pragma unroll
      for (int r = 0; r < 16; ++r)
        if (i0 + r < t.b) update1(a, c, ew + r, g[r]);
    }
  }

  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, s_bad != 0, s_t_enter, s_t_ready);
}

__global__ void __launch_bounds__(HD_THREADS, 1) v2_ps_hadamard_kernel(const PsArgs2 a) { ps_hadamard(a); }
__global__ void __launch_bounds__(HD_THREADS, 1) v2_ps_hadamard_lw_kernel(const PsArgsLw a) { ps_hadamard(a); }
__global__ void __launch_bounds__(HD_THREADS, 1) v2_ps_hadamard_gather_kernel(const PsArgsGather a) { ps_hadamard(a); }
__global__ void __launch_bounds__(HD_THREADS, 1) v2_ps_hadamard_lion_kernel(const PsArgsLion a) { ps_hadamard(a); }

// ---- --code-stats ------------------------------------------------------------------------------------------
struct HStatArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  int tile0;                   // global index of tiles[0] (partials are indexed by global encode tile)
  const long long* gptr;
  float* const* arena_peer;    // [n_owners] arena base inside each owner (this worker's (lo, step))
  int n_owners;
  long long arena_floats;
  int worker;
  const Ctrl2* ctrl;
  double* partials;            // [n_enc_tiles][STAT_PART]
  unsigned int* unit_counters; // [n_hadamard_units]
  double* acc;                 // [n_hadamard_units][STAT_ACC]
};

__global__ void __launch_bounds__(HD_THREADS) v2_hadamard_code_stats_kernel(const HStatArgs a) {
  __shared__ __align__(16) float s_x[HD_TILE];
  __shared__ double red[2][HD_WARPS];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  if (u.kind != KIND_HADAMARD) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int jt = t.owner;
  const float* slot = a.arena_peer[(u.own0 + jt) % a.n_owners] + (long long)a.worker * a.arena_floats + u.slot_off;
  const int d = u.K, levels = 1 << u.I;
  const int kb0 = t.a / d, nbt = (t.b + d - 1) / d;
  const int i0 = 16 * tid, kb = i0 / d;
  const long long e0 = (long long)t.a + i0;
  const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a;
  const int nch = (reinterpret_cast<uintptr_t>(src) & 15) == 0 ? (t.b >> 3) : 0;
  float x[16], v[16];
  hd_rotate(src, nch, t.b, e0, a.ctrl->seed, t.unit, a.ctrl->step, d, s_x, x, v);
  double gsq = 0.0, mse = 0.0;
  if (kb < nbt) {
    const long long poff = hd_params_off(u.n_ps) + 2LL * (kb0 + kb);
    const float lo = ld_cg_f(slot + poff), st = ld_cg_f(slot + poff + 1);
    const int nb = min(d, t.b - kb * d);
    const double w = (double)nb / ((double)d * (double)d) * (double)st * (double)st;
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const double xd = (double)x[r];
      gsq = fma(xd, xd, gsq);
      if (!(st > 0.f)) continue;
      const float tt = hd_t(v[r], lo, st);
      const float fl = floorf(tt);
      const double f = fl < (float)(levels - 1) ? (double)__fsub_rn(tt, fl) : 0.0;
      mse = fma(f * (1.0 - f), w, mse);
    }
    if (!(st >= 0.f) && (i0 & (d - 1)) == 0) mse += (double)st;   // special bucket: NaN
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
    for (int w = 0; w < HD_WARPS; ++w) { g += red[0][w]; m += red[1][w]; }
    stat_store_tile(a, u, g, m, (double)t.b, 0.0, (double)t.b, s_last);   // every element is an atom
  }
  __syncthreads();
  if (!s_last || tid != 0) return;
  double sum[STAT_PART];
  stat_unit_sum(a, u, sum);
  stat_accumulate(a, u, sum);
}

extern "C" {

void atomo_v2_launch_hadamard_encode(const void* units, const void* tiles, int tile0, int ntiles,
                                     const long long* gptr, float* const* arena_peer, int* const* sig_peer,
                                     int n_owners, long long arena_floats, int worker, int group, const void* ctrl,
                                     unsigned int* group_counter, long long* tstats, int final_group, float* residual,
                                     cudaStream_t stream) {
  if (ntiles <= 0) return;
  PushArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.tstats = tstats; a.final_group = final_group; a.residual = residual;
  if (residual != nullptr) v2_hadamard_encode_ef_kernel<<<ntiles, HD_THREADS, 0, stream>>>(a);
  else v2_hadamard_encode_kernel<<<ntiles, HD_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_hadamard(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks,
                                 int group, int final_group, int owner, float* master, float* mom, float* sq,
                                 float* sqmax, float* vmom, float* vsq, float* vsqmax, void* wshadow_mc,
                                 void* const* wshadow_peer, float* vparams_local, float* vparams_mc,
                                 float* const* vparams_peer, const float* vgrads_mc, const float* const* vgrads_peer,
                                 const float* arenas, long long arena_floats, int* sig, int* const* sig_peer,
                                 void* ctrl, unsigned int* group_counter, long long timeout, long long* tstats,
                                 float inv_w, int grid, cudaStream_t stream) {
  v2_ps_hadamard_kernel<<<ps_grid(grid, ntiles), HD_THREADS, 0, stream>>>(
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, final_group, owner, master, mom, sq, sqmax, vmom, vsq,
              vsqmax, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, vgrads_mc, vgrads_peer,
              nullptr, arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w));
}

void atomo_v2_launch_hadamard_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                         const long long* gptr, float* const* arena_peer, int n_owners,
                                         long long arena_floats, int worker, const void* ctrl, double* partials,
                                         unsigned int* unit_counters, double* acc, cudaStream_t stream) {
  if (ntiles <= 0) return;
  HStatArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr;
  a.arena_peer = arena_peer; a.n_owners = n_owners; a.arena_floats = arena_floats; a.worker = worker;
  a.ctrl = (const Ctrl2*)ctrl; a.partials = partials; a.unit_counters = unit_counters; a.acc = acc;
  v2_hadamard_code_stats_kernel<<<ntiles, HD_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_hadamard_lw(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLw& a = *static_cast<const PsArgsLw*>(args);
  v2_ps_hadamard_lw_kernel<<<ps_grid(grid, a.ntiles), HD_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_hadamard_gather(const void* args, int grid, cudaStream_t stream) {
  const PsArgsGather& a = *static_cast<const PsArgsGather*>(args);
  v2_ps_hadamard_gather_kernel<<<ps_grid(grid, a.ntiles), HD_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_hadamard_lion(const void* args, int grid, cudaStream_t stream) {
  const PsArgsLion& a = *static_cast<const PsArgsLion*>(args);
  v2_ps_hadamard_lion_kernel<<<ps_grid(grid, a.ntiles), HD_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
