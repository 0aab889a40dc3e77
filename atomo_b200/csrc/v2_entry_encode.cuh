// The encode body shared by the entry codes of the bf16 engine (v2_entrywise.cu: sampled entry-wise ATOMO,
// v2_topk.cu: deterministic top-k).  One CTA per tile (= one destination owner): the thread's 16 consecutive bf16
// elements are loaded, a compile-time keep policy decides which of them travel and which carry the exact flag, the
// optional error-feedback epilogue updates the residual, and the kept entries are compacted in element order by a
// warp + block scan (no atomics), staged in shared memory and stored into the owner's arena as 4-byte words, then
// count / scale and the tile's step stamp; the last CTA of the launch publishes flag[group][worker] = step on every
// owner.
//
// The keep decision is a compile-time policy (EntryKeep): KEEP_SAMPLE draws element i with probability
// p_i = min(1, |g_i| * s / L1) and flags p_i == 1 as exact (entry-wise ATOMO); KEEP_TOPK keeps the unit's k largest
// magnitudes (topk_keep, v2_topk.cu), all exact, with a header scale of 0.
#pragma once
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

constexpr int EE_THREADS = 256;
constexpr int EE_WARPS = EE_THREADS / 32;
constexpr int EE_PER_THREAD = ENTRY_TILE_ELEMS / EE_THREADS;   // 16 consecutive elements per thread
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

struct EEncArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  const long long* gptr;       // gradient base pointers (bf16), one per weight tensor
  const double* l1;            // entry-wise: per entry unit (v2_entry_stats_kernel)
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

// The uniform of element e of a unit is word (e & 3) of Philox(seed', counter = (e >> 2, unit, step, worker)):
// one Philox call serves 4 consecutive elements.  The seed differs from the QSGD rounding's.
__device__ __forceinline__ void entry_philox(const EEncArgs& a, int unit, long long e, int step, uint32_t (&r4)[4]) {
  Philox::gen(a.ctrl->seed ^ 0xd1b54a32d192ed03ULL, (uint32_t)(e >> 2), (uint32_t)unit, (uint32_t)step,
              (uint32_t)a.worker, r4);
}

enum EntryKeep : int { KEEP_SAMPLE = 0, KEEP_TOPK = 1 };
// top-k: the encode arguments plus the selection state, and the keep decision of the thread's 16 elements (both in
// v2_topk.cu, the only user)
struct TEncArgs;
__device__ __forceinline__ uint32_t topk_keep(const TEncArgs& a, const Tile2& t, const Unit2& u, const uint32_t (&h)[8]);

// Error feedback: what element x of A is owed after this push, x - g_hat (the owner's decode of the tile)
__device__ __forceinline__ float entry_residual(uint32_t bits, uint32_t kept, uint32_t exact, float scale) {
  const float x = __uint_as_float(bits << 16);
  return kept ? (exact ? 0.f : x - copysignf(scale, x)) : x;
}

template <int KEEP, bool EF, class Args>
__device__ __forceinline__ void entry_encode(const Args& a) {
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
  // Top-k: no norm, scale 0.
  const double L1 = KEEP == KEEP_TOPK ? 0.0 : a.l1[u.ts_index], s = (double)u.budget;
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
  if constexpr (KEEP == KEEP_TOPK) {
    keep = exact = topk_keep(a, t, u, h);
  } else {
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
        a.tstats[5] += now - a.tstats[9 + a.group];      // selection / stats + encode of this group
        if (a.final_group) a.tstats[8] += now - a.tstats[6];          // step start -> last push published
      }
    }
  }
}

}  // namespace v2
}  // namespace atomo
