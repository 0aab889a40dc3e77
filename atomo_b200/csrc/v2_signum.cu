// Signum with majority vote (Bernstein et al., ICML 2018 / ICLR 2019) and Distributed Lion (Liu et al., NeurIPS 2024) on
// the overlapped, sharded bf16 engine (sm_90a): the worker-side momentum, 1-bit encode and push of ONE backward group,
// and the owner-side vote (or mean) and step.  The oracles are codings/signum.py and codings/dlion.py.
//
//   v2_signum_encode_kernel  blocks [0, ntiles): one CTA per PS tile (one bucket of at most 4096 elements, one
//                            destination owner), 16 consecutive elements per thread.  The bf16 gradient g is read in
//                            place (16-byte loads where aligned); with beta > 0 the worker's fp32 momentum becomes
//                            u = beta u + g in place (float4, mc_step of v2_momentum.cuh), with beta == 0 u = g and no
//                            buffer exists.  Bit i of word j is element 64 j + i: 1 for u < 0, 0 for u > 0, and a fair
//                            Philox coin for u == 0 (+0, -0 and subnormals, which the fast-math arithmetic treats as
//                            zero).  Four threads make one 64-bit word; the words of the tile's real elements go into
//                            the owner's arena (the sign slot), then the bucket's status word (0, or NaN when some u of
//                            the tile is NaN / Inf) and the tile's step stamp.
//                            blocks [ntiles, ntiles + nv): the group's vector chunks, u = beta u + v in place in vmom
//                            and vgrads (the owners read vgrads).  The last CTA of the launch, tile or vector, publishes
//                            flag[group][worker] = step.  The group's only launch.  Bandwidth bound: 2 bytes read, 4 + 4
//                            read and written per weight element, 1/8 byte pushed.
//   v2_dlion_encode_kernel   the same launch with Lion's two-beta worker rule (v2_momentum.cuh) in place of
//                            the heavy-ball one: the bit is the sign of c = b1 m + (1 - b1) g, then m = b2 m + (1 - b2) g;
//                            vgrads receives c and vmom m.  With b1 == 0, c = g: no buffer and no vector chunks.
//   v2_ps_signum_kernel      one launch per (group, owner): the push wait / --num-aggregate mask and the stale-slot
//                            check of v2_ps_common.cuh.  Per weight tile and element, the 1 bits (neg) of the counted
//                            workers are summed by per-thread counters, pos = counted - neg, and
//                            vote = +1 (pos > neg), -1 (neg > pos), 0 (tie); a counted worker whose status word is not 0
//                            makes the tile's vote NaN.  p = fmaf(-lr, vote, p) through the SGD epilogue with momentum
//                            and weight decay 0, then the bf16 broadcast.  Vector tiles vote the same way on the sign of
//                            every counted worker's fp32 vgrads value, zeros by the same coin, any NaN / Inf value making
//                            the tile's vote NaN.
//   v2_ps_signum_mean_kernel the same launch with Distributed Lion's mean in place of the vote:
//                            v = (pos - neg) / counted (one rounded division; 0 when nothing is counted).
#include "v2_entry_encode.cuh"
#include "v2_momentum.cuh"

namespace atomo {
namespace v2 {

constexpr int SG_THREADS = 256;
constexpr int SG_TILE_ELEMS = 4096;
constexpr int SG_PER_THREAD = SG_TILE_ELEMS / SG_THREADS;
static_assert(SG_PER_THREAD == 16, "a thread holds 16 elements: a quarter of one 64-bit word");
constexpr unsigned long long SIGNUM_SEED_XOR = 0x9e6c63d0676a9a99ULL;   // the coin's own Philox key

// 0: positive, 1: negative, 2: zero (+-0 and subnormals), 3: NaN / Inf; decided on the bits, so that the class does not
// depend on how the compiler's flush-to-zero treats a comparison
__device__ __forceinline__ uint32_t signum_class(float x) {
  const uint32_t b = __float_as_uint(x), ex = b & 0x7f800000u;
  return ex == 0x7f800000u ? 3u : (ex == 0u ? 2u : (b >> 31));
}

// The coin of element e of a unit: word (e & 3) of Philox(seed', counter = (e >> 2, unit, step, worker)) as a uniform,
// 1 below one half.  The layout of entry_philox with a seed of its own.
__device__ __forceinline__ uint32_t signum_coin(unsigned long long seed, int unit, long long e, int step, int worker) {
  uint32_t r4[4];
  Philox::gen(seed ^ SIGNUM_SEED_XOR, (uint32_t)(e >> 2), (uint32_t)unit, (uint32_t)step, (uint32_t)worker, r4);
  const uint32_t r = (e & 2) ? ((e & 1) ? r4[3] : r4[2]) : ((e & 1) ? r4[1] : r4[0]);
  return Philox::to_uniform(r) < 0.5f ? 1u : 0u;
}

// the bit of a value of class cls (signum_class): its sign bit, or the coin for a zero
__device__ __forceinline__ uint32_t signum_bit(float x, uint32_t cls, uint32_t coin) {
  return cls == 2u ? coin : (__float_as_uint(x) >> 31);
}

__device__ __forceinline__ float signum_vote(int pos, int neg) {
  return pos > neg ? 1.f : (neg > pos ? -1.f : 0.f);
}

// the owners' aggregate of pos positive and neg negative signs: the vote, or (MEAN) their mean, 0 when nothing is counted
template <bool MEAN>
__device__ __forceinline__ float signum_aggregate(int pos, int neg) {
  if constexpr (MEAN)
    return pos + neg == 0 ? 0.f : __fdiv_rn((float)(pos - neg), (float)(pos + neg));
  else
    return signum_vote(pos, neg);
}

struct SignumEncArgs : PushArgs {
  int ntiles;                  // blocks [0, ntiles) are PS tiles, the rest vector chunks
  const EfChunk* vchunks;      // the group's vector chunks (plan2.vec_chunks), or nullptr
  float* mom;                  // worker momentum indexed like wshadow, or nullptr (beta == 0)
  float* vgrads;
  float* vmom;                 // worker momentum indexed like vgrads
  float beta;                  // Distributed Lion: b1
  const float* ext_uniforms;   // tests: uniforms indexed like wshadow, replacing the coin's Philox
};

struct DlionEncArgs : SignumEncArgs {
  float b2;
};

// The worker rules: the direction whose sign is pushed, from the gradient g and the worker's momentum m (updated in place)
struct HeavyBallRule {         // Signum: u = beta u + g, the direction is u
  float beta;
  __device__ __forceinline__ float operator()(float g, float& m) const { return mc_step(g, m, beta, false); }
};
struct LionRule {              // Distributed Lion: c = b1 m + (1 - b1) g, then m = b2 m + (1 - b2) g
  float b1, b2;
  __device__ __forceinline__ float operator()(float g, float& m) const {
    const float c = lion_direction(g, m, b1);
    m = lion_momentum(g, m, b2);
    return c;
  }
};

template <class Rule>
__device__ __forceinline__ void signum_encode_tile(const SignumEncArgs& a, int step, const Rule& rule) {
  const Tile2 t = a.tiles[blockIdx.x];
  const Unit2 u = a.units[t.unit];
  const int tid = threadIdx.x, lane = tid & 31;
  const int jt = t.owner;                                   // encode tiles: index of the tile inside its unit
  const int owner = (u.own0 + jt) % a.n_owners;
  float* slot = a.arena_peer[owner] + (long long)a.worker * a.arena_floats + u.slot_off;
  unsigned long long* words =
      reinterpret_cast<unsigned long long*>(slot + qsgd_words_off(u.n_ps, u.rows)) + (long long)jt * u.cols;
  const int i0 = tid * SG_PER_THREAD;
  const int n = t.b - i0;                                   // elements of this thread (<= 0: none, >= 16: 16)
  const long long e0 = (long long)t.a + i0;                 // element index inside the unit (a multiple of 16)
  uint32_t h[8];
  entry_load16(reinterpret_cast<const __nv_bfloat16*>(a.gptr[u.pidx]) + u.g_off + e0, n, h);
  float x[SG_PER_THREAD];
#pragma unroll
  for (int i = 0; i < SG_PER_THREAD; ++i) x[i] = __uint_as_float(bf16_bits(h, i) << 16);
  if (a.mom != nullptr && n > 0) {
    float* up = a.mom + u.w_off + e0;                       // 64-byte aligned: w_off % 64 == 0, e0 % 16 == 0
    if (n >= SG_PER_THREAD) {
#pragma unroll
      for (int j = 0; j < SG_PER_THREAD / 4; ++j) {
        float4 v = reinterpret_cast<const float4*>(up)[j];
        x[4 * j] = rule(x[4 * j], v.x);
        x[4 * j + 1] = rule(x[4 * j + 1], v.y);
        x[4 * j + 2] = rule(x[4 * j + 2], v.z);
        x[4 * j + 3] = rule(x[4 * j + 3], v.w);
        reinterpret_cast<float4*>(up)[j] = v;
      }
    } else {
#pragma unroll
      for (int i = 0; i < SG_PER_THREAD; ++i) {
        if (i < n) {
          float ui = up[i];
          x[i] = rule(x[i], ui);
          up[i] = ui;
        }
      }
    }
  }
  uint32_t bits = 0;
  int bad = 0;
#pragma unroll
  for (int i = 0; i < SG_PER_THREAD; ++i) {
    if (i < n) {
      const uint32_t cls = signum_class(x[i]);
      uint32_t coin = 0;
      if (cls == 2u)
        coin = a.ext_uniforms != nullptr ? (a.ext_uniforms[u.w_off + e0 + i] < 0.5f ? 1u : 0u)
                                         : signum_coin(a.ctrl->seed, t.unit, e0 + i, step, a.worker);
      bits |= signum_bit(x[i], cls, coin) << i;
      bad |= cls == 3u;
    }
  }
  // thread tid holds bits 16 (tid & 3) .. + 15 of word tid >> 2; only the words of real elements are stored
  unsigned long long w = (unsigned long long)bits << (16 * (lane & 3));
  w |= __shfl_xor_sync(0xffffffffu, w, 1);
  w |= __shfl_xor_sync(0xffffffffu, w, 2);
  if ((lane & 3) == 0 && (tid >> 2) < ((t.b + 63) >> 6)) words[tid >> 2] = w;
  const int nonfinite = __syncthreads_or(bad);

  // ---- the bucket's status word and the tile's step stamp (after its words), then the group's push flag ----------
  if (tid == 0) {
    slot[qsgd_norms_off(u.n_ps) + jt] = nonfinite ? __int_as_float(0x7fffffff) : 0.f;
    enc_stamp(reinterpret_cast<int*>(slot), jt, step);
    enc_push_flag(a, step);
  }
}

template <class Rule>
__device__ __forceinline__ void signum_encode(const SignumEncArgs& a, const Rule& rule) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && a.tstats != nullptr) a.tstats[9 + a.group] = globaltimer_ns();
  const int step = a.ctrl->step;
  if ((int)blockIdx.x < a.ntiles) {
    signum_encode_tile(a, step, rule);
    return;
  }
  const EfChunk c = a.vchunks[blockIdx.x - a.ntiles];
  float* s = a.vgrads + c.w_off + c.start;
  float* um = a.vmom + c.w_off + c.start;
  for (int i = threadIdx.x; i < c.count; i += blockDim.x) {
    float ui = um[i];
    s[i] = rule(s[i], ui);
    um[i] = ui;
  }
  __syncthreads();
  if (threadIdx.x == 0) enc_push_flag(a, step);
}

__global__ void __launch_bounds__(SG_THREADS) v2_signum_encode_kernel(const SignumEncArgs a) {
  signum_encode(a, HeavyBallRule{a.beta});
}

__global__ void __launch_bounds__(SG_THREADS) v2_dlion_encode_kernel(const DlionEncArgs a) {
  signum_encode(a, LionRule{a.beta, a.b2});
}

// ---- PS: vote + step --------------------------------------------------------------------------------------------
struct SignumPsArgs : PsArgs2 {
  const float* vext;          // tests: the coins' uniforms of the vector elements, [worker][vparams index], or nullptr
  long long vext_stride;
};

// the vote (or mean) of a vector tile into OUT (NaN everywhere when a counted value is not finite), then the step and
// the fp32 broadcast
template <bool MEAN>
__device__ __forceinline__ void signum_vec_tile(const SignumPsArgs& a, const OptC& c, const Unit2& u, const Tile2& t,
                                                int unit, unsigned int wmask, int step, float* OUT) {
  const int tid = threadIdx.x;
  const long long e0 = u.w_off + t.a;
  const unsigned long long seed = a.ctrl->seed;
  int bad = 0;
  __syncthreads();   // previous tile is done with OUT
  for (int i = tid; i < t.b; i += blockDim.x) {
    int neg = 0, cnt = 0;
    for (int w = 0; w < a.W; ++w) {
      if (!((wmask >> w) & 1u)) continue;
      const float x = ld_cg_f(a.vgrads_peer[w] + e0 + i);
      const uint32_t cls = signum_class(x);
      uint32_t coin = 0;
      if (cls == 2u)
        coin = a.vext != nullptr ? (a.vext[w * a.vext_stride + e0 + i] < 0.5f ? 1u : 0u)
                                 : signum_coin(seed, unit, (long long)t.a + i, step, w);
      neg += (int)signum_bit(x, cls, coin);
      bad |= cls == 3u;
      ++cnt;
    }
    OUT[i] = signum_aggregate<MEAN>(cnt - neg, neg);
  }
  const int nonfinite = __syncthreads_or(bad);
  for (int i = tid; i < t.b; i += blockDim.x) {
    const long long e = e0 + i;
    float p = a.vparams_local[e], m = 0.f, q = 0.f, qm = 0.f;
    opt_update(nonfinite ? __int_as_float(0x7fffffff) : OUT[i], p, m, q, qm, c);
    for (int r = 0; r < a.nranks; ++r) a.vparams_peer[r][e] = p;
  }
}

template <bool MEAN>
__device__ __forceinline__ void ps_signum(const SignumPsArgs& a) {
  __shared__ __align__(16) float OUT[SG_TILE_ELEMS];   // the votes of one tile, physical element order
  __shared__ int s_ok, s_bad, s_nf;
  __shared__ unsigned int s_mask, s_use;
  __shared__ long long s_t_enter, s_t_ready;
  const int tid = threadIdx.x;
  Ctrl2* ctrl = a.ctrl;
  const int step = ctrl->step;

  ps_wait(a, ctrl, step, s_ok, s_bad, s_mask, s_t_enter, s_t_ready);
  const bool ok = s_ok != 0;
  const unsigned int wmask = s_mask;
  // the step is p - lr vote (or mean): the momentum lives on the workers, and the weight decay is v2_decay's launch before this one
  OptC c = ps_opt_consts(ctrl, step);
  c.opt = OPT_SGD; c.mu = 0.f; c.wd = 0.f;
  const auto [t_begin, t_end] = ps_tile_range(a);
  for (int ti = t_begin; ok && ti < t_end; ++ti) {
    const Tile2 t = a.tiles[ti];
    const Unit2 u = a.units[t.unit];
    if (u.kind == KIND_VEC) {
      signum_vec_tile<MEAN>(a, c, u, t, t.unit, wmask, step, OUT);
      continue;
    }
    if (u.kind != KIND_SIGNUM) continue;
    const int jt = t.a / u.ps_rows;
    const long long soff = qsgd_norms_off(u.n_ps), woff = qsgd_words_off(u.n_ps, u.rows);
    __syncthreads();   // previous tile is done with OUT / s_use / s_nf
    if (tid == 0) {
      const unsigned int use = ps_fresh_workers(a, u, jt, wmask, step, s_bad);
      int nf = 0;
      for (int w = 0; w < a.W; ++w)
        if ((use >> w) & 1u) nf |= ld_cg_f(a.arenas + (long long)w * a.arena_floats + u.slot_off + soff + jt) != 0.f;
      s_use = use;
      s_nf = nf;
    }
    __syncthreads();
    const unsigned int use = s_use;
    // thread tid: elements 16 tid .. 16 tid + 15 of the tile, the 16-bit half (tid & 1) of int32 word tid >> 1
    const int i0 = tid * SG_PER_THREAD;
    if (i0 < t.b) {
      int neg[SG_PER_THREAD];
#pragma unroll
      for (int i = 0; i < SG_PER_THREAD; ++i) neg[i] = 0;
      for (int w = 0; w < a.W; ++w) {
        if (!((use >> w) & 1u)) continue;
        const int* hw = reinterpret_cast<const int*>(a.arenas + (long long)w * a.arena_floats + u.slot_off + woff) +
                        2LL * jt * u.cols;
        const uint32_t b = ((uint32_t)ld_cg_i(hw + (tid >> 1))) >> (16 * (tid & 1));
#pragma unroll
        for (int i = 0; i < SG_PER_THREAD; ++i) neg[i] += (int)((b >> i) & 1u);
      }
      const int counted = __popc(use);
      const bool nf = s_nf != 0;
#pragma unroll
      for (int i = 0; i < SG_PER_THREAD; ++i)
        if (i0 + i < t.b)
          OUT[i0 + i] = nf ? __int_as_float(0x7fffffff) : signum_aggregate<MEAN>(counted - neg[i], neg[i]);
    }
    __syncthreads();
    // fused SGD epilogue + bf16 parameter broadcast
    const long long e0 = u.w_off + t.a;
    const int nvec = ((e0 & 7) == 0) ? (t.b >> 3) : 0;
    for (int v = tid; v < nvec; v += blockDim.x) {
      const float4 g0 = *reinterpret_cast<const float4*>(&OUT[8 * v]);
      const float4 g1 = *reinterpret_cast<const float4*>(&OUT[8 * v + 4]);
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      update8(a, c, e0 + 8LL * v, g);
    }
    for (int i = (nvec << 3) + tid; i < t.b; i += blockDim.x) update1(a, c, e0 + i, OUT[i]);
  }

  __syncthreads();
  if (tid == 0) ps_complete(a, ctrl, step, s_bad != 0, s_t_enter, s_t_ready);
}

__global__ void __launch_bounds__(SG_THREADS) v2_ps_signum_kernel(const SignumPsArgs a) { ps_signum<false>(a); }

__global__ void __launch_bounds__(SG_THREADS) v2_ps_signum_mean_kernel(const SignumPsArgs a) { ps_signum<true>(a); }

extern "C" {

void atomo_v2_launch_signum_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                   const void* vchunks, int nv, float* vgrads, float* mom, float* vmom, float beta,
                                   float* const* arena_peer, int* const* sig_peer, int n_owners,
                                   long long arena_floats, int worker, int group, const void* ctrl,
                                   unsigned int* group_counter, long long* tstats, int final_group,
                                   const float* ext_uniforms, cudaStream_t stream) {
  if (ntiles + nv <= 0) return;
  SignumEncArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.tstats = tstats; a.final_group = final_group; a.residual = nullptr;
  a.ntiles = ntiles; a.vchunks = (const EfChunk*)vchunks; a.mom = mom; a.vgrads = vgrads; a.vmom = vmom; a.beta = beta;
  a.ext_uniforms = ext_uniforms;
  v2_signum_encode_kernel<<<ntiles + nv, SG_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_dlion_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                  const void* vchunks, int nv, float* vgrads, float* mom, float* vmom, float b1,
                                  float b2, float* const* arena_peer, int* const* sig_peer, int n_owners,
                                  long long arena_floats, int worker, int group, const void* ctrl,
                                  unsigned int* group_counter, long long* tstats, int final_group,
                                  const float* ext_uniforms, cudaStream_t stream) {
  if (ntiles + nv <= 0) return;
  DlionEncArgs a;
  a.units = (const Unit2*)units; a.tiles = (const Tile2*)tiles + tile0; a.gptr = gptr;
  a.arena_peer = arena_peer; a.sig_peer = sig_peer; a.n_owners = n_owners; a.arena_floats = arena_floats;
  a.worker = worker; a.group = group; a.ctrl = (const Ctrl2*)ctrl; a.group_counter = group_counter;
  a.tstats = tstats; a.final_group = final_group; a.residual = nullptr;
  a.ntiles = ntiles; a.vchunks = (const EfChunk*)vchunks; a.mom = mom; a.vgrads = vgrads; a.vmom = vmom; a.beta = b1;
  a.b2 = b2; a.ext_uniforms = ext_uniforms;
  v2_dlion_encode_kernel<<<ntiles + nv, SG_THREADS, 0, stream>>>(a);
}

void atomo_v2_launch_ps_signum(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks,
                               int group, int final_group, int owner, float* master, float* mom, float* sq,
                               float* sqmax, float* vmom, float* vsq, float* vsqmax, void* wshadow_mc,
                               void* const* wshadow_peer, float* vparams_local, float* vparams_mc,
                               float* const* vparams_peer, const float* vgrads_mc, const float* const* vgrads_peer,
                               const float* arenas, long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                               unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                               const float* vext, long long vext_stride, int mean, cudaStream_t stream) {
  SignumPsArgs a;
  static_cast<PsArgs2&>(a) =
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, final_group, owner, master, mom, sq, sqmax, vmom, vsq,
              vsqmax, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, vgrads_mc, vgrads_peer,
              nullptr, arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats, inv_w);
  a.vext = vext;
  a.vext_stride = vext_stride;
  if (mean)
    v2_ps_signum_mean_kernel<<<ps_grid(grid, ntiles), SG_THREADS, 0, stream>>>(a);
  else
    v2_ps_signum_kernel<<<ps_grid(grid, ntiles), SG_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
