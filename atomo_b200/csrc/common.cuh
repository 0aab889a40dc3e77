// Shared device helpers for the atomo_b200 sm_90a kernels.
//
// * system-scope acquire/release accessors used for cross-GPU flags living in
//   NVLink peer memory (the replacement for the reference's MPI tag handshakes,
//   SURVEY.md 2.6 C1/C2/C6),
// * NVLS multicast accessors (multimem.st / multimem.ld_reduce),
// * Philox4x32-10 counter-based RNG (replacement for np.random.binomial /
//   np.random.rand in codings/svd.py:61 and codings/qsgd.py:63),
// * the layer/tile descriptor tables every grouped kernel walks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace atomo {

// SMs of the current device: the grid caps of the grid-stride launches are a few resident CTAs per SM
// (132 on an H100 SXM).  Queried once per process; an engine process drives one device.
inline int num_sms() {
  static int n = 0;
  if (n < 1) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n < 1) n = 132;
  }
  return n;
}

// ----------------------------------------------------------------------------
// Descriptor tables (built once on the host by runtime/engine.py, resident in HBM)
// ----------------------------------------------------------------------------
enum Route : int { ROUTE_DENSE = 0, ROUTE_SVD_TS = 1, ROUTE_LOWRANK_EXT = 2 };

struct LayerDesc {
  long long off;         // element offset of the tensor in the flat fp32 param/grad buffers
  long long slot_off;    // float offset of this layer's slot inside one worker arena (low-rank routes)
  long long gpart_off;   // float offset of this layer's Gram partials (ntiles x cols*cols)
  int numel;             // elements of the tensor
  int rows;              // tall dimension M of the matricized gradient
  int cols;              // skinny dimension n (<= 64 for ROUTE_SVD_TS)
  int row_stride;        // element stride between tall rows      (A[r][c] = base[off + r*row_stride + c*col_stride])
  int col_stride;        // element stride between skinny columns
  int route;             // Route
  int rcap;              // slot capacity in atoms (multiple of 4)
  int ts_index;          // index among ROUTE_SVD_TS layers (gram partial / selection scratch), else -1
  int tile0;             // first entry of this layer in the encode tile table
  int ntiles;            // number of encode tiles
  int vec_ok;            // 1 when flat float4 access is legal (contiguous layout, 16B-aligned tiles)
  int ps_rows;           // rows per PS tile
};

// slot layout inside a worker arena, in floats, starting at LayerDesc::slot_off:
//   [0..3]   header: {count (int), step (int), 0, 0}
//   [4 .. 4+rcap)                 s[a]        = sigma_a / p_a
//   [4+rcap .. 4+rcap+rcap*cols)  V[a][c]     (row a = right singular vector, length cols)
//   [...   .. +rows*rcap)         U[r][a]     (row-major, stride rcap)
__host__ __device__ inline long long slot_s_off() { return 4; }
__host__ __device__ inline long long slot_v_off(int rcap) { return 4 + rcap; }
__host__ __device__ inline long long slot_u_off(int rcap, int cols) {
  long long o = 4 + (long long)rcap + (long long)rcap * cols;
  return (o + 3) & ~3LL;  // keep U 16-byte aligned
}
__host__ __device__ inline long long slot_floats(int rows, int cols, int rcap) {
  long long o = slot_u_off(rcap, cols) + (long long)rows * rcap;
  return (o + 31) & ~31LL;  // 128-byte aligned slots
}

struct TileDesc {
  int layer;  // index into the LayerDesc table
  int row0;   // first tall row of the tile (dense route: first element / 4)
  int nrows;  // rows in this tile         (dense route: number of elements)
  int col0;   // first column (column-tiled wide layers), else 0
};

constexpr int RCAP_MAX = 32;     // max atoms per slot
constexpr int TS_MAX_COLS = 64;  // widest skinny dimension the Gram/Jacobi path handles

// Per-rank control block (device memory).  Everything a CUDA-graph replay must
// see change lives here, not in kernel arguments.
struct Ctrl {
  int step;            // current global step (starts at 1 like STEP_START_)
  int error;           // sticky error code (spin-wait timeouts etc.)
  float lr;            // learning rate (host updates on the LR schedule)
  float momentum;
  float dampening;
  float weight_decay;
  int nesterov;
  int first_step;      // step at which momentum buffers are initialised (buf = g)
  unsigned long long seed;
  unsigned int done_encode;   // CTA-completion counters (self-resetting)
  unsigned int done_ps;
  unsigned int done_aux;
  unsigned int pad;
};

enum ErrorCode : int { ERR_NONE = 0, ERR_WAIT_PUSH_TIMEOUT = 1, ERR_WAIT_PARAM_TIMEOUT = 2, ERR_SLOT_OVERFLOW = 3 };

// ----------------------------------------------------------------------------
// memory-model helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_relaxed_sys(const int* p) {
  int v;
  asm volatile("ld.relaxed.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_na_f4(float4* p, const float4 v) {  // streaming store (peer/HBM)
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}
__device__ __forceinline__ float4 ld_nc_f4(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
// volatile-ish (L2-coherent) loads for data another GPU just wrote into our HBM
__device__ __forceinline__ float4 ld_cg_f4(const float4* p) {
  float4 v;
  asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_cg_f(const float* p) {
  float v;
  asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ int ld_cg_i(const int* p) {
  int v;
  asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

// NVLS multicast: one store replicated by the switch to every GPU of the group
__device__ __forceinline__ void multimem_st_f4(float4* mc, const float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void multimem_st_i(int* mc, int v) {
  asm volatile("multimem.st.release.sys.global.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}
// NVLS in-switch reduction: load the SUM over every GPU's copy
__device__ __forceinline__ float4 multimem_ld_reduce_f4(const float4* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}

__device__ __forceinline__ long long globaltimer_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Bounded spin on a step-stamped flag written by a peer GPU.  Returns false on
// timeout (caller records an error instead of hanging the GPU forever).
__device__ __forceinline__ bool spin_wait_ge(const int* flag, int want, long long max_ns) {
  long long t0 = clock64();
  // clock64 ticks at SM clock (~1-2 GHz): treat ticks as ~ns, a 2x error is irrelevant for a timeout
  int backoff = 32;
  while (ld_acquire_sys(flag) < want) {
    __nanosleep(backoff);
    if (backoff < 1024) backoff <<= 1;
    if (clock64() - t0 > max_ns) return false;
  }
  return true;
}

// ----------------------------------------------------------------------------
// warp / block reductions
// ----------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ----------------------------------------------------------------------------
// Philox4x32-10
// ----------------------------------------------------------------------------
struct Philox {
  static constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
  __host__ __device__ static inline void round(uint32_t (&c)[4], uint32_t (&k)[2]) {
#ifdef __CUDA_ARCH__
    uint32_t hi0 = __umulhi(M0, c[0]), hi1 = __umulhi(M1, c[2]);
#else
    uint32_t hi0 = (uint32_t)(((uint64_t)M0 * c[0]) >> 32), hi1 = (uint32_t)(((uint64_t)M1 * c[2]) >> 32);
#endif
    uint32_t lo0 = M0 * c[0], lo1 = M1 * c[2];
    uint32_t n0 = hi1 ^ c[1] ^ k[0], n1 = lo1, n2 = hi0 ^ c[3] ^ k[1], n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k[0] += W0; k[1] += W1;
  }
  // 4 x 32 random bits for (key=seed, counter=(c0,c1,c2,c3))
  __host__ __device__ static inline void gen(unsigned long long seed, uint32_t c0, uint32_t c1, uint32_t c2,
                                             uint32_t c3, uint32_t (&out)[4]) {
    uint32_t c[4] = {c0, c1, c2, c3};
    uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
#pragma unroll
    for (int i = 0; i < 10; ++i) round(c, k);
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
  }
  __host__ __device__ static inline float to_uniform(uint32_t x) {  // [0,1)
    return (float)(x >> 8) * (1.0f / 16777216.0f);
  }
};

}  // namespace atomo
