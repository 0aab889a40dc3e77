// Top-k sparsification on the overlapped, sharded bf16 engine (sm_90a): every >= 2-D weight is one entry unit
// (the slots, tiles and PS of entry-wise ATOMO, v2_entrywise.cu) whose k = budget largest-magnitude entries are pushed
// exactly.  Magnitudes are compared on the bf16 bits (bits & 0x7fff orders finite magnitudes exactly); entries of
// magnitude 0 are never kept; entries equal to the threshold T are kept in increasing element order until k_eff =
// min(k, nnz) are kept; a tensor with an Inf or NaN keeps nothing.  Everything is integer counting, so the kept set
// has the same bits on every run, and no launch needs the host or a memset (the per-unit state resets itself).
//
//   v2_topk_hist_kernel     one CTA per encode tile: a shared 256-bin histogram of the magnitudes' bits 14..7,
//                           added into the unit's histogram; the unit's last tile (unit counter) takes the histogram
//                           (clearing it), scans it from the top and finds the bin B holding the k_eff-th magnitude.
//   v2_topk_refine_kernel   one CTA per encode tile: a 128-bin histogram of bits 6..0 of the magnitudes in bin B,
//                           kept per tile and added into the unit's histogram; the unit's last tile finds T and
//                           need_ties = k_eff - #(> T).
//   v2_topk_encode_kernel   entry_encode (v2_entry_encode.cuh) with the top-k keep policy: |g| > T, or |g| == T with a
//                           tie rank (T counts of the unit's earlier tiles + in-tile prefix) below need_ties; every
//                           kept entry carries the exact flag, the header's scale is 0.  The owners decode with
//                           v2_ps_entry_kernel unchanged.  v2_topk_encode_ef_kernel adds the error-feedback epilogue,
//                           v2_topk_encode_mc_kernel also momentum-factor masking (momentum correction, v2_momentum.cu).
//   v2_topk_code_stats_kernel  --code-stats of top-k units, in the layout of v2_code_stats_kernel (v2_stats.cu).
#include "v2_entry_encode.cuh"

namespace atomo {
namespace v2 {

struct TSelArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  int tile0;                   // global index of tiles[0] (tile counts are indexed by global encode tile)
  const long long* gptr;
  int* hist;                   // [n_entry_units][TOPK_HI_BINS], zero between launches
  int* tile_counts;            // [n_enc_tiles][TOPK_LO_BINS]
  unsigned int* unit_counters; // [n_entry_units]
  int* sel;                    // [n_entry_units][TOPK_STATE]
  long long* tstats;
  int group;
};

// Sum of c over threads tid..255 of the block (bins at and above bin tid): warp suffix scan, then the warp totals.
__device__ __forceinline__ int block_suffix_sum(int c, int* wtot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_down_sync(0xffffffffu, incl, o);
    if (lane + o < 32) incl += v;
  }
  if (lane == 0) wtot[warp] = incl;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < EE_WARPS; ++w)
    if (w > warp) incl += wtot[w];
  return incl;
}

// Add the tile's bins into the unit's histogram, then count the tile; true in the unit's last tile, whose CTA then
// sees every tile's additions.
__device__ __forceinline__ bool topk_publish(const TSelArgs& a, const Unit2& u, int c, int* s_last) {
  if (c) atomicAdd(a.hist + TOPK_HI_BINS * u.ts_index + threadIdx.x, c);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int old = atomicAdd(&a.unit_counters[u.ts_index], 1u);
    *s_last = (old == (unsigned int)u.n_enc - 1u) ? 1 : 0;
    if (*s_last) a.unit_counters[u.ts_index] = 0;
  }
  __syncthreads();
  if (!*s_last) return false;
  __threadfence();
  return true;
}

__global__ void __launch_bounds__(EE_THREADS) v2_topk_hist_kernel(const TSelArgs a) {
  __shared__ int sh[TOPK_HI_BINS];
  __shared__ int wtot[EE_WARPS];
  __shared__ int s_last, s_total, s_bad;
  static_assert(TOPK_HI_BINS == EE_THREADS, "one bin per thread");
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x;
  if (blockIdx.x == 0 && tid == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();
  sh[tid] = 0;
  __syncthreads();
  const int i0 = tid * EE_PER_THREAD;
  uint32_t h[8];
  entry_load16(reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a + i0, t.b - i0, h);
#pragma unroll
  for (int i = 0; i < EE_PER_THREAD; ++i) {
    const uint32_t m = bf16_bits(h, i) & 0x7fffu;      // elements past the tile's end read as 0
    if (m) atomicAdd(&sh[m >> 7], 1);
  }
  __syncthreads();
  if (!topk_publish(a, u, sh[tid], &s_last)) return;

  int* uh = a.hist + TOPK_HI_BINS * u.ts_index;
  const int c = atomicExch(uh + tid, 0);                  // take the unit's histogram, leave it zero
  const int S = block_suffix_sum(c, wtot);                // non-zero magnitudes in bins >= tid
  if (tid == 0) s_total = S;
  if (tid == TOPK_HI_BINS - 1) s_bad = c;                 // bin 255: exponent all ones, Inf / NaN
  __syncthreads();
  const int k = (int)u.budget;
  const int keff = s_bad ? 0 : min(k, s_total);
  int* st = a.sel + TOPK_STATE * u.ts_index;
  if (keff == 0) {
    if (tid == 0) {
      st[TK_BIN] = -1; st[TK_NEED_BIN] = 0; st[TK_T] = TOPK_NONE; st[TK_NEED_TIES] = 0; st[TK_KEFF] = 0;
      st[TK_NONFINITE] = s_bad ? 1 : 0;
    }
  } else if (S - c < keff && keff <= S) {                 // exactly one bin: the one holding the k_eff-th magnitude
    st[TK_BIN] = tid; st[TK_NEED_BIN] = keff - (S - c); st[TK_T] = TOPK_NONE; st[TK_NEED_TIES] = 0;
    st[TK_KEFF] = keff; st[TK_NONFINITE] = 0;
  }
}

__global__ void __launch_bounds__(EE_THREADS) v2_topk_refine_kernel(const TSelArgs a) {
  __shared__ int sh[TOPK_LO_BINS];
  __shared__ int wtot[EE_WARPS];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x;
  int* st = a.sel + TOPK_STATE * u.ts_index;
  const int B = st[TK_BIN];
  if (tid < TOPK_LO_BINS) sh[tid] = 0;
  __syncthreads();
  if (B >= 0) {
    const int i0 = tid * EE_PER_THREAD;
    uint32_t h[8];
    entry_load16(reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + t.a + i0, t.b - i0, h);
#pragma unroll
    for (int i = 0; i < EE_PER_THREAD; ++i) {
      const uint32_t m = bf16_bits(h, i) & 0x7fffu;
      if (m && (int)(m >> 7) == B) atomicAdd(&sh[m & 127u], 1);
    }
  }
  __syncthreads();
  int c = 0;
  if (tid < TOPK_LO_BINS) {
    c = sh[tid];
    a.tile_counts[(long long)TOPK_LO_BINS * (a.tile0 + blockIdx.x) + tid] = c;   // the tie counts of the encode
  }
  if (!topk_publish(a, u, c, &s_last)) return;

  int* uh = a.hist + TOPK_HI_BINS * u.ts_index;
  c = tid < TOPK_LO_BINS ? atomicExch(uh + tid, 0) : 0;
  const int S = block_suffix_sum(c, wtot);
  const int need = st[TK_NEED_BIN];
  if (B >= 0 && S - c < need && need <= S) {
    st[TK_T] = (B << 7) | tid;
    st[TK_NEED_TIES] = need - (S - c);
  }
}

// ---- encode: entry_encode (v2_entry_encode.cuh) with the top-k keep policy ---------------------------------------
struct TEncArgs : EEncArgs {
  const int* sel;              // [n_entry_units][TOPK_STATE] (v2_topk_refine_kernel)
  const int* tile_counts;      // [n_enc_tiles][TOPK_LO_BINS]
};

// Kept: |g| > T, or |g| == T with a tie rank below need_ties.  The rank of a tie counts the T entries of the unit's
// earlier tiles, then those of the tile before it in element order (thread order: a thread holds 16 consecutive
// elements).  Elements past the tile's end read as 0 and are never kept.
__device__ __forceinline__ uint32_t topk_keep(const TEncArgs& a, const Tile2& t, const Unit2& u, const uint32_t (&h)[8]) {
  __shared__ int s_ties[EE_WARPS], s_base[EE_WARPS];
  const int* st = a.sel + TOPK_STATE * u.ts_index;
  const int T = st[TK_T], need = st[TK_NEED_TIES];
  uint32_t keep = 0, eq = 0;
#pragma unroll
  for (int i = 0; i < EE_PER_THREAD; ++i) {
    const int m = (int)(bf16_bits(h, i) & 0x7fffu);
    if (m > T) keep |= 1u << i;
    else if (m == T) eq |= 1u << i;
  }
  if (need > 0) {                                         // the same for every thread of the CTA (one unit)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int b = 0;
    for (int j = tid; j < t.owner; j += EE_THREADS)       // encode tiles: t.owner = index of the tile in its unit
      b += a.tile_counts[(long long)TOPK_LO_BINS * (u.enc_tile0 + j) + (T & (TOPK_LO_BINS - 1))];
    const int c = __popc(eq);
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
      b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane == 31) s_ties[warp] = incl;
    if (lane == 0) s_base[warp] = b;
    __syncthreads();
    int rank = incl - c;
#pragma unroll
    for (int w = 0; w < EE_WARPS; ++w) {
      rank += s_base[w];
      if (w < warp) rank += s_ties[w];
    }
#pragma unroll
    for (int i = 0; i < EE_PER_THREAD; ++i) {
      if ((eq >> i) & 1u) {
        if (rank < need) keep |= 1u << i;
        ++rank;
      }
    }
  }
  return keep;
}

__global__ void __launch_bounds__(EE_THREADS) v2_topk_encode_kernel(const TEncArgs a) {
  entry_encode<KEEP_TOPK, false>(a);
}
// error feedback: the same encode plus the residual epilogue (kept entries are exact: residual 0, others keep A_i)
__global__ void __launch_bounds__(EE_THREADS) v2_topk_encode_ef_kernel(const TEncArgs a) {
  entry_encode<KEEP_TOPK, true>(a);
}
// momentum correction: the error-feedback encode, and the worker's momentum zeroed at every kept entry
__global__ void __launch_bounds__(EE_THREADS) v2_topk_encode_mc_kernel(const TEncArgs a, float* mom) {
  entry_encode<KEEP_TOPK, true, true>(a, mom);
}

// ---- --code-stats for top-k units ----------------------------------------------------------------------------
// The partials / accumulator layout of every --code-stats kernel (STAT_PART / STAT_ACC, v2_common.cuh).  gsq = ||bf16(g)||^2; mse = the dropped energy, the entries below T plus the
// tile's dropped ties times T^2 (the convention of svd top-k); expected atoms = k_eff, realized = the header counts.
struct TStatArgs {
  const Unit2* units;
  const Tile2* tiles;          // already offset to the first tile of the group
  int tile0;                   // global index of tiles[0]
  const long long* gptr;
  const int* sel;
  const int* tile_counts;
  float* const* arena_peer;    // [n_owners] arena base inside each owner (this worker's tile headers)
  int n_owners;
  long long arena_floats;
  int worker;
  double* partials;            // [n_enc_tiles][STAT_PART]
  unsigned int* unit_counters; // [n_entry_units]
  double* acc;                 // [n_entry_units][STAT_ACC]
};

__global__ void __launch_bounds__(EE_THREADS) v2_topk_code_stats_kernel(const TStatArgs a) {
  __shared__ double red[2][EE_WARPS];
  __shared__ int red_above[EE_WARPS];
  __shared__ int s_last;
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  if (u.kind != KIND_ENTRY) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int jt = t.owner;
  const int* st = a.sel + TOPK_STATE * u.ts_index;
  const int T = st[TK_T];
  const unsigned short* src = reinterpret_cast<const unsigned short*>(a.gptr[u.pidx]) + u.g_off + t.a;
  double gsq = 0.0, mse = 0.0;
  int above = 0;
  for (int i = tid; i < t.b; i += EE_THREADS) {
    const uint32_t b = src[i];
    const double x = (double)__uint_as_float(b << 16), x2 = x * x;
    const int m = (int)(b & 0x7fffu);
    gsq += x2;
    if (m < T) mse += x2;
    else if (m > T) ++above;                              // kept
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    gsq += __shfl_xor_sync(0xffffffffu, gsq, o);
    mse += __shfl_xor_sync(0xffffffffu, mse, o);
    above += __shfl_xor_sync(0xffffffffu, above, o);
  }
  if (lane == 0) { red[0][warp] = gsq; red[1][warp] = mse; red_above[warp] = above; }
  __syncthreads();
  if (tid == 0) {
    double g = 0.0, m = 0.0;
    int ab = 0;
    for (int w = 0; w < EE_WARPS; ++w) { g += red[0][w]; m += red[1][w]; ab += red_above[w]; }
    const float* slot = a.arena_peer[(u.own0 + jt) % a.n_owners] + (long long)a.worker * a.arena_floats + u.slot_off;
    const int real = ld_cg_i(reinterpret_cast<const int*>(slot + entry_hdr_off(jt)) + 1);
    const int ties = T < TOPK_NONE
        ? a.tile_counts[(long long)TOPK_LO_BINS * (a.tile0 + blockIdx.x) + (T & (TOPK_LO_BINS - 1))] : 0;
    const double tv = (double)__uint_as_float((uint32_t)T << 16);
    // the tile's store and the unit's sum stay inline: as helpers they change this kernel's register allocation
    double* p = a.partials + (long long)STAT_PART * (a.tile0 + blockIdx.x);
    p[0] = g;
    p[1] = m + (double)(ties - (real - ab)) * tv * tv;    // ties not kept
    p[2] = 0.0;
    p[3] = 0.0;
    p[4] = (double)real;
    __threadfence();
    const unsigned int old = atomicAdd(&a.unit_counters[u.ts_index], 1u);
    s_last = (old == (unsigned int)u.n_enc - 1u) ? 1 : 0;
    if (s_last) a.unit_counters[u.ts_index] = 0;
  }
  __syncthreads();
  if (!s_last || tid != 0) return;
  __threadfence();
  double sum[STAT_PART] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < u.n_enc; ++k) {                     // tile order: the same bits on every run
    const double* pk = a.partials + (long long)STAT_PART * (u.enc_tile0 + k);
    for (int f = 0; f < STAT_PART; ++f) sum[f] += __ldcg(pk + f);
  }
  sum[2] = (double)st[TK_KEFF];
  double* acc = a.acc + (long long)STAT_ACC * u.ts_index;
  for (int f = 0; f < STAT_PART; ++f) acc[f] += sum[f];
  acc[5] += sum[4];
  acc[6] += 1.0;
}

extern "C" {

int atomo_v2_topk_state_ints() { return TOPK_STATE; }
int atomo_v2_topk_hist_bins() { return TOPK_HI_BINS; }
int atomo_v2_topk_tile_bins() { return TOPK_LO_BINS; }

void atomo_v2_launch_topk_select(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 int* hist, int* tile_counts, unsigned int* unit_counters, int* sel, long long* tstats,
                                 int group, cudaStream_t stream) {
  if (ntiles <= 0) return;
  TSelArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr;
  a.hist = hist; a.tile_counts = tile_counts; a.unit_counters = unit_counters; a.sel = sel; a.tstats = tstats;
  a.group = group;
  v2_topk_hist_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a);
  v2_topk_refine_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_topk_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 const int* sel, const int* tile_counts, float* const* arena_peer,
                                 int* const* sig_peer, int n_owners, long long arena_floats, int worker, int group,
                                 const void* ctrl, unsigned int* group_counter, long long* tstats, int final_group,
                                 float* residual, float* mom, cudaStream_t stream) {
  if (ntiles <= 0) return;
  TEncArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr; a.l1 = nullptr;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.ext_uniforms = nullptr; a.tstats = tstats; a.final_group = final_group; a.residual = residual;
  a.sel = sel; a.tile_counts = tile_counts;
  if (mom != nullptr) v2_topk_encode_mc_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a, mom);
  else if (residual != nullptr) v2_topk_encode_ef_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a);
  else v2_topk_encode_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_topk_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                     const long long* gptr, const int* sel, const int* tile_counts,
                                     float* const* arena_peer, int n_owners, long long arena_floats, int worker,
                                     double* partials, unsigned int* unit_counters, double* acc, cudaStream_t stream) {
  if (ntiles <= 0) return;
  TStatArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.tile0 = tile0; a.gptr = gptr; a.sel = sel;
  a.tile_counts = tile_counts; a.arena_peer = arena_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.partials = partials; a.unit_counters = unit_counters; a.acc = acc;
  v2_topk_code_stats_kernel<<<ntiles, EE_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
