// Grouped skinny GEMM on the Hopper tensor cores (warpgroup MMA, `wgmma.mma_async`), sm_90a.
//
// The subspace-iteration route of the spectral coder needs, for every square-ish layer
// (fc, 1x1 convolutions), products with a skinny right-hand side of width l = 16/32:
//     Y = A X      (m x n)(n x l)        "forward":  M = m, K = n
//     B = A^T Q    (n x m)(m x l)        "backward": M = n, K = m
// They are bandwidth-bound on reading the fp32 gradient A exactly once per product — provided the
// 2*m*n*l FLOPs do not land on the CUDA cores.  This kernel walks a table of 128-row output tiles
// (all layers in one launch): every CTA (one warpgroup) stages K-chunks of A and of the skinny operand in
// shared memory in the canonical no-swizzle K-major GMMA layout (8 x 16-byte core matrices), the warpgroup
// issues `wgmma.mma_async.m64nNk8.f32.tf32.tf32` for the two 64-row halves of the tile with the fp32
// accumulators in registers, and a 2-stage pipeline refills the other stage (and has the global loads of
// the chunk after that in flight) while the tensor core consumes the current one.  The epilogue writes the
// accumulator fragments straight from registers to the m x l result.
#include "common.cuh"

namespace atomo {

struct GemmTile {
  const float* A;   // element (i, k) of the M x K operand at A[i * sa_i + k * sa_k]
  const float* B;   // element (j, k) of the N x K operand at B[j * sb_j + k * sb_k]
  float* C;         // element (i, j) of the M x N result at C[i * ldc + j]
  int sa_i, sa_k, sb_j, sb_k;
  int ldc, M, N, K;  // M <= 128 valid rows in this tile, N in {16, 32}
  int a_vec;         // 1: float4 along k legal, 2: float4 along i legal, 0: scalar gather
  int k_begin;       // split-K: this tile reduces k in [k_begin, k_begin + k_len)   (k_len == 0 -> whole K)
  int k_len;
  int atomic;        // 1: accumulate into C with atomicAdd (split-K partial sums; C pre-zeroed)
};

constexpr int GEMM_THREADS = 128;           // one warpgroup
constexpr int GEMM_KC = 32;                 // K chunk per stage (tf32: 4 MMAs of K = 8)
constexpr int GEMM_LBO = 144;               // bytes between core matrices adjacent in K (padded: fewer bank conflicts)
constexpr int GEMM_SBO = GEMM_LBO * (GEMM_KC / 4);   // bytes between 8-row groups
constexpr int GEMM_A_STAGE = 16 * GEMM_SBO; // 128 rows
constexpr int GEMM_B_STAGE = 4 * GEMM_SBO;  // up to 32 rows

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  // GMMA shared-memory matrix descriptor (PTX ISA, "Matrix Descriptor Format" of wgmma): start>>4 [0,14),
  // leading byte offset (between core matrices adjacent in K)>>4 [16,30), stride byte offset (between 8-row
  // groups)>>4 [32,46), base_offset=0 [49,52), layout_type=no swizzle (0) [62,64)
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((GEMM_LBO >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((GEMM_SBO >> 4) & 0x3FFF) << 32;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D (64 x N, fp32, registers) += A (64 x 8, smem) * B (N x 8, smem)^T, both operands K-major tf32
__device__ __forceinline__ void wgmma_tf32(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc)
      : "memory");
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc)
      : "memory");
}

// one element (row i, reduction index k) of a staged operand, canonical K-major no-swizzle layout
__device__ __forceinline__ uint32_t core_off(int i, int k) {
  return (uint32_t)((i >> 3) * GEMM_SBO + (k >> 2) * GEMM_LBO + (i & 7) * 16 + (k & 3) * 4);
}

template <int N>
__device__ __forceinline__ void gemm_tile(const GemmTile& T, unsigned char* const (&sA)[2],
                                          unsigned char* const (&sB)[2]) {
  const int tid = threadIdx.x;
  const int kb = T.k_begin;
  const int kend = T.k_len > 0 ? min(T.K, kb + T.k_len) : T.K;
  const int nchunks = (kend - kb + GEMM_KC - 1) / GEMM_KC;

  // register staging: the global loads of chunk kc+1 are issued before the MMAs of chunk kc-1 are waited for,
  // so DRAM latency overlaps the tensor-core work and the shared-memory hand-off
  float ra[32];
  float rb[8];
  auto load_regs = [&](int k0) {
    if (T.a_vec == 1) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int e = tid + q * GEMM_THREADS;
        const int i = e >> 3, k = k0 + 4 * (e & 7);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < T.M && k < kend) {
          const float* src = T.A + (long long)i * T.sa_i + k;
          if (k + 3 < kend) v = __ldg(reinterpret_cast<const float4*>(src));
          else { v.x = __ldg(src); if (k + 1 < kend) v.y = __ldg(src + 1); if (k + 2 < kend) v.z = __ldg(src + 2); }
        }
        ra[4 * q] = v.x; ra[4 * q + 1] = v.y; ra[4 * q + 2] = v.z; ra[4 * q + 3] = v.w;
      }
    } else if (T.a_vec == 2) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int e = tid + q * GEMM_THREADS;
        const int kk = e >> 5, i = 4 * (e & 31), k = k0 + kk;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < kend && i < T.M) {
          const float* src = T.A + i + (long long)k * T.sa_k;
          if (i + 3 < T.M) v = __ldg(reinterpret_cast<const float4*>(src));
          else { v.x = __ldg(src); if (i + 1 < T.M) v.y = __ldg(src + 1); if (i + 2 < T.M) v.z = __ldg(src + 2); }
        }
        ra[4 * q] = v.x; ra[4 * q + 1] = v.y; ra[4 * q + 2] = v.z; ra[4 * q + 3] = v.w;
      }
    } else {
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        const int e = tid + q * GEMM_THREADS;
        const int i = e >> 5, k = k0 + (e & 31);
        ra[q] = (i < T.M && k < kend) ? __ldg(T.A + (long long)i * T.sa_i + (long long)k * T.sa_k) : 0.f;
      }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int e = tid + q * GEMM_THREADS;
      float v = 0.f;
      if (e < N * GEMM_KC) {
        int j, kk;
        if (T.sb_k == 1) { j = e >> 5; kk = e & 31; }
        else { kk = e / N; j = e - kk * N; }
        const int k = k0 + kk;
        if (k < kend) v = __ldg(T.B + (long long)j * T.sb_j + (long long)k * T.sb_k);
      }
      rb[q] = v;
    }
  };
  auto store_regs = [&](int s) {
    if (T.a_vec == 1) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int e = tid + q * GEMM_THREADS;
        *reinterpret_cast<float4*>(sA[s] + core_off(e >> 3, 4 * (e & 7))) =
            make_float4(ra[4 * q], ra[4 * q + 1], ra[4 * q + 2], ra[4 * q + 3]);
      }
    } else if (T.a_vec == 2) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int e = tid + q * GEMM_THREADS;
        const int kk = e >> 5, i = 4 * (e & 31);
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<float*>(sA[s] + core_off(i + j, kk)) = ra[4 * q + j];
      }
    } else {
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        const int e = tid + q * GEMM_THREADS;
        *reinterpret_cast<float*>(sA[s] + core_off(e >> 5, e & 31)) = ra[q];
      }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int e = tid + q * GEMM_THREADS;
      if (e < N * GEMM_KC) {
        int j, kk;
        if (T.sb_k == 1) { j = e >> 5; kk = e & 31; }
        else { kk = e / N; j = e - kk * N; }
        *reinterpret_cast<float*>(sB[s] + core_off(j, kk)) = rb[q];
      }
    }
  };

  // accumulators of the two 64-row halves: fragment element r of thread (warp w, lane l) is row
  // 16 w + l/4 + 8 ((r/2) & 1), column 8 (r/4) + 2 (l & 3) + (r & 1) of its half
  float acc[2][N / 2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int r = 0; r < N / 2; ++r) acc[h][r] = 0.f;

  // Stage s = kc & 1 is rewritten at chunk kc + 2.  The MMAs of chunk kc are waited for (by every warp) before
  // the barrier of chunk kc + 1, so that rewrite is ordered after them; the MMAs of chunk kc overlap the
  // shared-memory stores and the global loads of the chunks after it.
  load_regs(kb);
  for (int kc = 0; kc < nchunks; ++kc) {
    const int s = kc & 1;
    store_regs(s);
    if (kc + 1 < nchunks) load_regs(kb + (kc + 1) * GEMM_KC);  // in flight across the wait, barrier and MMAs
    wgmma_wait_all();                                           // chunk kc-1 has been consumed
    // generic-proxy writes -> visible to the tensor core's async proxy
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    wgmma_fence();
    const uint32_t a0 = smem_u32(sA[s]), b0 = smem_u32(sB[s]);
#pragma unroll
    for (int ks = 0; ks < GEMM_KC / 8; ++ks) {
      const uint64_t bdesc = make_smem_desc(b0 + ks * 2 * GEMM_LBO);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        wgmma_tf32(acc[h], make_smem_desc(a0 + h * 8 * GEMM_SBO + ks * 2 * GEMM_LBO), bdesc);
    }
    wgmma_commit();
  }
  wgmma_wait_all();

  // ---- epilogue: accumulator fragments -> C ---------------------------------------------------------------
  const int warp = tid >> 5, lane = tid & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int q = 0; q < N / 4; ++q) {
      const int i = h * 64 + warp * 16 + (lane >> 2) + 8 * (q & 1);
      const int j = 8 * (q >> 1) + 2 * (lane & 3);
      if (i >= T.M) continue;
      float* dst = T.C + (long long)i * T.ldc + j;
      const float v0 = acc[h][2 * q], v1 = acc[h][2 * q + 1];
      if (T.atomic) {
        atomicAdd(dst, v0);  // split-K partial sum
        atomicAdd(dst + 1, v1);
      } else if ((((uintptr_t)dst) & 7) == 0) {
        *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
      } else {
        dst[0] = v0;
        dst[1] = v1;
      }
    }
  }
  // the next tile's stores reuse both stages: every warp is past this tile's MMAs (waited above)
  __syncthreads();
}

__global__ void __launch_bounds__(GEMM_THREADS)
skinny_gemm_tf32_kernel(const GemmTile* __restrict__ tiles, int ntiles, Ctrl* ctrl) {
  extern __shared__ __align__(128) unsigned char gsm[];
  unsigned char* const sA[2] = {gsm, gsm + GEMM_A_STAGE};
  unsigned char* const sB[2] = {gsm + 2 * GEMM_A_STAGE, gsm + 2 * GEMM_A_STAGE + GEMM_B_STAGE};
  for (int ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
    const GemmTile T = tiles[ti];
    if (T.N == 16) gemm_tile<16>(T, sA, sB);
    else if (T.N == 32) gemm_tile<32>(T, sA, sB);
    else if (threadIdx.x == 0) atomicExch(&ctrl->error, 4 /* malformed tile: N not in {16, 32} */);
  }
}

extern "C" {
int atomo_gemm_tile_bytes() { return (int)sizeof(GemmTile); }
int atomo_gemm_smem_bytes() { return 2 * GEMM_A_STAGE + 2 * GEMM_B_STAGE; }

void atomo_launch_skinny_gemm(const void* tiles, int ntiles, void* ctrl, int grid, cudaStream_t stream) {
  if (ntiles <= 0) return;
  static bool attr_set = false;
  const int smem = atomo_gemm_smem_bytes();
  if (!attr_set) {
    cudaFuncSetAttribute(skinny_gemm_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr_set = true;
  }
  if (grid < 1) grid = 1;
  if (grid > ntiles) grid = ntiles;
  skinny_gemm_tf32_kernel<<<grid, GEMM_THREADS, smem, stream>>>((const GemmTile*)tiles, ntiles, (Ctrl*)ctrl);
}
}
}  // namespace atomo
