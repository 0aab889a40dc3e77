// Descriptor tables + helpers of the overlapped / sharded bf16 engine (kernels v2_encode.cu, v2_ps.cu;
// host planner ops/plan2.py — the struct layouts below are mirrored there byte for byte).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace atomo {
namespace v2 {

enum Kind : int {
  KIND_SLAB = 1, KIND_MAT = 2, KIND_DENSE16 = 3, KIND_VEC = 4, KIND_QSGD = 5, KIND_ENTRY = 6, KIND_SIGN = 7,
  KIND_POWER = 8, KIND_FP8 = 9
};

// One coding unit: a conv gradient in [O][K][I] (channels_last) layout ("SLAB": row (o,ri), column (b,k) of the
// reference's (O*I/2, 2K) matricization is X_o[k][2ri+b]), a <=64-column block of a 2-D matrix ("MAT"), or a
// dense chunk (bf16 weight sent dense / fp32 vector).
//
// QSGD / TernGrad units ("QSGD", v2_qsgd.cu: one per >= 2-D weight, buckets over the physical element order) reuse
// the fields:  K = bucket (elements), I = q (quantization level), rows = buckets, cols = L (uint64 words per
// bucket), rs = 1 for TernGrad (0 for QSGD), cs = buckets per PS tile, ps_rows = elements per PS tile,
// ts_index = index among the QSGD units (TernGrad clip / stats counter).
//
// Scaled-sign units ("SIGN", v2_sign.cu: one per >= 2-D weight) use the QSGD fields and slot with one bit per element:
// K = bucket, rows = buckets, cols = L = ceil(bucket / 64) uint64 words per bucket, cs = buckets per PS tile,
// ps_rows = elements per PS tile, ts_index = index among the sign units; the slot's norms are the fp32 scales.
//
// FP8 units ("FP8", v2_fp8.cu) have the fields and slot of the sign units with one e4m3 byte per element:
// cols = ceil(bucket / 8) uint64 words per bucket, the bytes in element order; the norms are the fp32 scales 2^-k.
//
// PowerSGD units ("POWER", v2_powersgd.cu: one per >= 2-D weight with r (O + C) < O C): rows = O, cols = C (row o is
// the contiguous physical slab of output channel o), rcap = r, K = pass-B column blocks, n_enc = pass-A row tiles,
// ps_rows = rows per PS tile, gpart_off = float offset of the worker-local factors and warm state, ts_index = index
// among the PowerSGD units (state / stats counter).
//
// Entry-wise units ("ENTRY", v2_entrywise.cu: one per >= 2-D weight, tiles over the physical element order) use
// budget = expected atoms s (clamped to [1, numel]), ps_rows = elements per tile (ENTRY_TILE_ELEMS),
// ts_index = index among the entry units (L1 norm / stats counter).
struct Unit2 {
  long long w_off;      // element offset of the unit's base in wshadow / master / momentum (VEC: in vparams)
  long long g_off;      // element offset inside the parameter's own gradient tensor
  long long slot_off;   // float offset of the unit's slot inside one worker arena
  long long gpart_off;  // float offset of the Gram partials (n_enc x cols*cols)
  int kind;
  int pidx;             // index into the gradient pointer table
  int rows, cols;       // tall matricized shape of the unit
  int K, I;             // SLAB: taps, input channels
  int rs, cs;           // MAT: element strides of rows / columns (DENSE16: rs = offset in the staging region)
  int rcap;             // slot capacity in atoms (multiple of 4)
  float budget;         // expected number of atoms (sparsity budget of this unit)
  int numel;
  int group;
  int enc_tile0, n_enc;
  int ps_rows;          // rows per PS tile
  int own0;             // owner of PS tile 0 (tile j -> (own0 + j) % n_owners)
  int ps_tile0, n_ps;
  int ts_index;         // index among coded units (vsel / selcount / counters)
  int ubits;            // 0: U fp32 [rows][rcap]; 8 (QSVD): U int8 [rows][rcap] + one fp32 scale per row
};
static_assert(sizeof(Unit2) == 112, "Unit2 layout must match ops/plan2.py UNIT_FMT");

struct Tile2 {
  int unit;
  int a;      // SLAB encode: first slab; MAT encode / PS low-rank: first row; dense: first element
  int b;      // count (slabs / rows / elements)
  int owner;
};

enum Opt : int { OPT_SGD = 0, OPT_ADAM = 1, OPT_AMSGRAD = 2 };

struct Ctrl2 {
  int step;
  int error;
  float lr, momentum, dampening, weight_decay;
  int nesterov;
  int first_step;
  unsigned long long seed;
  float beta1, beta2, eps, pad0;
  int opt;
  int num_aggregate;   // 0 = wait for every worker; N = proceed after N pushes (backup workers)
  int pad1, pad2;
};
static_assert(sizeof(Ctrl2) == 72, "Ctrl2 layout must match ops/plan2.py CTRL2_FMT");

enum Err2 : int { ERR2_NONE = 0, ERR2_WAIT_PUSH = 1, ERR2_WAIT_PARAM = 2, ERR2_SLOT_STEP = 4, ERR2_NONFINITE = 8 };

constexpr int MAX_WORKERS = 16;
constexpr int MAX_GROUPS = 8;
constexpr int V2_MAX_COLS = TS_MAX_COLS;
constexpr int V2_RCAP_MAX = RCAP_MAX;
// signal region (ints): push flag of (group g, worker w) at g*MAX_WORKERS + w; param flag of owner o at 256 + o;
// aggregation mask of (group g) at 320 + g (owner-local)
constexpr int SIG_PUSH = 0;
constexpr int SIG_PARAM = 256;
constexpr int SIG_MASK = 320;

__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

// ---- mbarrier / TMA 1-D bulk copy ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "V2_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra V2_DONE;\n"
      "bra V2_WAIT;\n"
      "V2_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// One SLAB encode tile = `ns` consecutive slabs = ns*K rows of I bf16 each.  Rows are copied by TMA bulk copies
// (one per row, issued by the 32 lanes of warp 0) into a row pitch of I/2 + 4 words, which makes both consumers
// bank-conflict free: the Gram's 4x4 register blocks read the same channel pair of different taps (stride = pitch,
// 4 words off a multiple of 32 banks), the projection reads 32 consecutive channel pairs of one tap.
__device__ __forceinline__ int slab_pitch_words(int I) { return (I >> 1) + 4; }

__device__ __forceinline__ void load_slab_tile(const __nv_bfloat16* gbase, int K, int I, int ns, uint32_t* sm,
                                               uint64_t* bar) {
  const int nrows = ns * K;
  const int pitch = slab_pitch_words(I);
  if (threadIdx.x < 32) {
    if (threadIdx.x == 0) mbar_expect_tx(bar, (uint32_t)nrows * I * 2);
    __syncwarp();
    for (int r = threadIdx.x; r < nrows; r += 32)
      bulk_g2s(sm + (size_t)r * pitch, gbase + (size_t)r * I, (uint32_t)I * 2, bar);
  }
}

// debugging / fallback path: the same tile through plain 16-byte loads (no TMA, no mbarrier)
__device__ __forceinline__ void load_slab_tile_ldg(const __nv_bfloat16* gbase, int K, int I, int ns, uint32_t* sm) {
  const int nrows = ns * K, pitch = slab_pitch_words(I), cpr = I >> 3;   // 16-byte chunks per row
  for (int idx = threadIdx.x; idx < nrows * cpr; idx += blockDim.x) {
    const int r = idx / cpr, c = idx - r * cpr;
    *reinterpret_cast<uint4*>(sm + (size_t)r * pitch + 4 * c) =
        __ldg(reinterpret_cast<const uint4*>(gbase + (size_t)r * I) + c);
  }
}

// slot layout (floats, from Unit2::slot_off inside one worker arena) — same as round 1:
//   [0..3] header {count, step, cols, rows} | s[rcap] | V[rcap][cols] | U[rows][rcap]
__host__ __device__ inline long long slot2_u_off(int rcap, int cols) {
  long long o = 4 + (long long)rcap + (long long)rcap * cols;
  return (o + 3) & ~3LL;
}
// QSVD slots: int8 U occupies rows*rcap/4 floats (rounded to 4), then rows fp32 scales (max |u| of the row)
__host__ __device__ inline long long slot2_scale_off(int rows, int rcap, int cols) {
  return slot2_u_off(rcap, cols) + (((long long)rows * rcap / 4 + 3) & ~3LL);
}

// QSGD slots (floats, from Unit2::slot_off inside one worker arena):
//   int32 step stamp per PS tile [n_ps, padded to 4] | fp32 bucket norms [rows, padded to 4] | uint64 words [rows][cols]
__host__ __device__ inline long long qsgd_norms_off(int n_ps) { return ((long long)n_ps + 3) & ~3LL; }
__host__ __device__ inline long long qsgd_words_off(int n_ps, int rows) {
  return qsgd_norms_off(n_ps) + (((long long)rows + 3) & ~3LL);
}

// Entry-wise slots (floats, from Unit2::slot_off inside one worker arena):
//   16-byte header per PS tile {int32 step stamp, int32 count, fp32 scale, pad} [n_ps] | per tile j, from
//   entry_words_off(n_ps, j, ps_rows): room for ps_rows uint32 entries (the last tile: its length rounded up to 4).
// Entry word: bits 0-11 element offset inside the tile, bit 12 set when p_i == 1 (the value is the bf16 gradient in
// bits 16-31), else the value is copysign(scale, bf16 gradient).
constexpr int ENTRY_TILE_ELEMS = 4096;
constexpr uint32_t ENTRY_FLAG_EXACT = 1u << 12;
__host__ __device__ inline long long entry_hdr_off(int j) { return 4LL * j; }
__host__ __device__ inline long long entry_words_off(int n_ps, int j, int ps_rows) {
  return 4LL * n_ps + (long long)j * ps_rows;
}

// Top-k entry units (v2_topk.cu; same slots, budget = k): the selection state of unit ts_index is
// sel[TOPK_STATE * ts_index + TK_*]; hist[TOPK_HI_BINS * ts_index] is the unit's histogram (all zero between launches),
// tiles[TOPK_LO_BINS * encode tile] the tile's counts of the low magnitude bits inside the threshold's high bin.
// A threshold of TOPK_NONE keeps nothing (all-zero or non-finite tensor).
constexpr int TOPK_STATE = 8;
constexpr int TOPK_HI_BINS = 256;     // magnitude bits 14..7
constexpr int TOPK_LO_BINS = 128;     // magnitude bits 6..0
constexpr int TOPK_NONE = 0x8000;
enum TopkField : int { TK_BIN = 0, TK_NEED_BIN = 1, TK_T = 2, TK_NEED_TIES = 3, TK_KEFF = 4, TK_NONFINITE = 5 };

}  // namespace v2
}  // namespace atomo
