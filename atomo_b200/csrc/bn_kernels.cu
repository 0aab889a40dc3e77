// Fused training-mode BatchNorm (+ residual add) (+ ReLU) for NHWC bf16 activations (sm_90a).
//
// ResNet-18 on 32x32 inputs is memory/latency bound: the stock path spends a large share of the
// step in batch_norm_collect_statistics / transform_input / backward_reduce / backward_elemt plus
// separate add and ReLU kernels.  Here the whole
//      y = relu( gamma * (x - mean) / sqrt(var + eps) + beta  [+ residual] )
// is two passes over x (statistics, then normalise+add+ReLU in one sweep) and the backward is two
// passes (per-channel reductions of dy*mask and dy*mask*xhat, then dx [+ d_residual] in one sweep).
// All tensors are viewed as [R = N*H*W][C] with C % 8 == 0; every access is a 16-byte vector of
// 8 bf16 channels; statistics are accumulated in fp32.
//
// With ReLU the forward also writes a 1-bit mask, uint8 [R][C/8]: bit i of byte e is (y > 0) for channel i of the
// bf16 vector y[e] it stored, so the backward reads 1 bit per element instead of re-reading y (2 bytes).
//
// Each layer runs two chains of three kernels (stats -> sum_partials -> apply, bwd_reduce -> sum_partials ->
// bwd_apply).  The second and third kernel of a chain are launched with programmatic dependent launch: their CTAs
// are scheduled while the predecessor drains, and they wait (griddepcontrol.wait) before any global read or write,
// so every result is the same as in plain stream order.  The first kernel of a chain follows a cuDNN kernel and
// is launched plainly.
#include <cuda_bf16.h>
#include <stdlib.h>

#include "common.cuh"

namespace atomo {

constexpr int BN_THREADS = 256;
constexpr int BN_MAX_C = 2048;

struct bf16x8 {
  uint4 v;
};

__device__ __forceinline__ void unpack8(const uint4 v, float (&f)[8]) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(p[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 v;
  __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

// programmatic dependent launch: wait until the previous kernel in the stream has completed and its writes are
// visible (a no-op in a plain launch) / allow the next kernel's CTAs to be scheduled from now on
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }

// The per-channel reductions are deterministic: every reduction CTA writes its partial sums to its own row of
// `part` ([gridDim.x][2C], no atomics) and bn_sum_partials_kernel adds the rows in a fixed order, so a step
// computes the same bits on every run.

// ---- pass 1 (forward): per-channel sum and sum of squares -------------------------------------------
// part row layout: [0..C) sum, [C..2C) sumsq
__global__ void __launch_bounds__(BN_THREADS)
bn_stats_kernel(const uint4* __restrict__ x, long long R, int C, float* __restrict__ part) {
  extern __shared__ float red[];  // [RL][C] x 2
  const int CG = C >> 3;
  const int RL = BN_THREADS / CG;
  const int cg = threadIdx.x % CG, rl = threadIdx.x / CG;
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
  if (rl < RL) {
    // 4 independent 16-byte loads in flight per thread: the per-layer tensors are 2-16 MB (L2 resident right
    // after the producing conv), so the kernel is latency bound unless every thread keeps several requests open
    const long long stride = (long long)gridDim.x * RL;
    long long r = (long long)blockIdx.x * RL + rl;
    for (; r + 3 * stride < R; r += 4 * stride) {
      uint4 v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = __ldg(x + (r + k * stride) * CG + cg);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float f[8];
        unpack8(v[k], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i] += f[i]; q[i] = fmaf(f[i], f[i], q[i]); }
      }
    }
    for (; r < R; r += stride) {
      float f[8];
      unpack8(__ldg(x + r * CG + cg), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) { s[i] += f[i]; q[i] = fmaf(f[i], f[i], q[i]); }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      red[rl * C + cg * 8 + i] = s[i];
      red[RL * C + rl * C + cg * 8 + i] = q[i];
    }
  }
  pdl_launch_dependents();
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int k = 0; k < RL; ++k) { a += red[k * C + c]; b += red[RL * C + k * C + c]; }
    part[(long long)blockIdx.x * 2 * C + c] = a;
    part[(long long)blockIdx.x * 2 * C + C + c] = b;
  }
}

// ---- pass 2 (forward): normalise + affine (+ residual) (+ ReLU and its mask); block 0 also finalises the statistics
__global__ void __launch_bounds__(BN_THREADS)
bn_apply_kernel(const uint4* __restrict__ x, const uint4* __restrict__ res, uint4* __restrict__ y,
                uint8_t* __restrict__ mask, long long R, int C, const float* __restrict__ acc,
                const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ save_mean,
                float* __restrict__ save_invstd, float* __restrict__ running_mean, float* __restrict__ running_var,
                float eps, float momentum, int relu) {
  extern __shared__ float tab[];  // scale[C], shift[C]
  pdl_wait();
  const float invR = 1.f / (float)R;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float mean = acc[c] * invR;
    const float v = acc[C + c] * invR - mean * mean;
    const float var = v < 0.f ? 0.f : v;  // not fmaxf: fmaxf(NaN, 0) = 0 would give a non-finite channel finite stats
    const float invstd = rsqrtf(var + eps);
    const float sc = gamma[c] * invstd;
    tab[c] = sc;
    tab[C + c] = beta[c] - mean * sc;
    if (blockIdx.x == 0) {
      save_mean[c] = mean;
      save_invstd[c] = invstd;
      if (running_mean != nullptr) {
        const float unbiased = R > 1 ? var * (float)R / (float)(R - 1) : var;
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
      }
    }
  }
  __syncthreads();
  const int CG = C >> 3;
  const long long total = R * CG;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(e % CG);
    float f[8], o[8];
    unpack8(__ldg(x + e), f);
    if (res != nullptr) {
      float g[8];
      unpack8(__ldg(res + e), g);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = fmaf(f[i], tab[cg * 8 + i], tab[C + cg * 8 + i]) + g[i];
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = fmaf(f[i], tab[cg * 8 + i], tab[C + cg * 8 + i]);
    }
    if (relu) {
      // a NaN stays NaN, as in stock ReLU (fmaxf(NaN, 0) is 0); every other o gets exactly fmaxf(o, 0)
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = o[i] != o[i] ? o[i] : fmaxf(o[i], 0.f);
    }
    const uint4 out = pack8(o);
    y[e] = out;
    if (relu) {
      // the bits come from the stored bf16 values (a positive fp32 o can round to bf16 zero), compared exactly as
      // the backward compared y before it read the mask; a NaN output passes its gradient, as stock
      // threshold_backward (y <= 0 ? 0 : dy) does
      float yv[8];
      unpack8(out, yv);
      unsigned m = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) m |= (!(yv[i] <= 0.f) ? 1u : 0u) << i;
      mask[e] = (uint8_t)m;
    }
  }
}

// ---- pass 1 (backward): per-channel sum(dy*mask) and sum(dy*mask*xhat) ------------------------------------------
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_reduce_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x, const uint8_t* __restrict__ mask,
                     long long R, int C, const float* __restrict__ mean, const float* __restrict__ invstd,
                     float* __restrict__ part, int relu) {
  extern __shared__ float red[];
  const int CG = C >> 3;
  const int RL = BN_THREADS / CG;
  const int cg = threadIdx.x % CG, rl = threadIdx.x / CG;
  float s[8], q[8], mu[8], is[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; mu[i] = mean[cg * 8 + i]; is[i] = invstd[cg * 8 + i]; }
  if (rl < RL) {
    const long long stride = (long long)gridDim.x * RL;
    long long r = (long long)blockIdx.x * RL + rl;
    for (; r + stride < R; r += 2 * stride) {   // 2 rows x 3 tensors = 6 independent loads in flight
      uint4 dv[2], xq[2];
      unsigned mq[2];
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        dv[k] = __ldg(dy + (r + k * stride) * CG + cg);
        xq[k] = __ldg(x + (r + k * stride) * CG + cg);
        if (relu) mq[k] = __ldg(mask + (r + k * stride) * CG + cg);
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        float d[8], xv[8];
        unpack8(dv[k], d);
        unpack8(xq[k], xv);
        if (relu) {
#pragma unroll
          for (int i = 0; i < 8; ++i) d[i] = (mq[k] >> i) & 1u ? d[i] : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i] += d[i]; q[i] = fmaf(d[i], (xv[i] - mu[i]) * is[i], q[i]); }
      }
    }
    for (; r < R; r += stride) {
      float d[8], xv[8];
      unpack8(__ldg(dy + r * CG + cg), d);
      unpack8(__ldg(x + r * CG + cg), xv);
      if (relu) {
        const unsigned m = __ldg(mask + r * CG + cg);
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = (m >> i) & 1u ? d[i] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) { s[i] += d[i]; q[i] = fmaf(d[i], (xv[i] - mu[i]) * is[i], q[i]); }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      red[rl * C + cg * 8 + i] = s[i];
      red[RL * C + rl * C + cg * 8 + i] = q[i];
    }
  }
  pdl_launch_dependents();
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int k = 0; k < RL; ++k) { a += red[k * C + c]; b += red[RL * C + k * C + c]; }
    part[(long long)blockIdx.x * 2 * C + c] = a;
    part[(long long)blockIdx.x * 2 * C + C + c] = b;
  }
}

// ---- pass 2 (backward): dx (and the masked dy for the residual branch); block 0 writes dgamma / dbeta ----------
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_apply_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x, const uint8_t* __restrict__ mask,
                    uint4* __restrict__ dx, uint4* __restrict__ dres, long long R, int C,
                    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                    const float* __restrict__ acc, float* __restrict__ dgamma, float* __restrict__ dbeta, int relu) {
  extern __shared__ float tab[];  // mean[C], invstd[C], a[C] = gamma*invstd, b[C] = sum_dy/R, c[C] = sum_dy_xhat/R
  pdl_wait();
  const float invR = 1.f / (float)R;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    tab[c] = mean[c];
    tab[C + c] = invstd[c];
    tab[2 * C + c] = gamma[c] * invstd[c];
    tab[3 * C + c] = acc[c] * invR;
    tab[4 * C + c] = acc[C + c] * invR;
    if (blockIdx.x == 0) {
      dbeta[c] = acc[c];
      dgamma[c] = acc[C + c];
    }
  }
  __syncthreads();
  const int CG = C >> 3;
  const long long total = R * CG;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(e % CG) * 8;
    float d[8], xv[8], o[8];
    unpack8(__ldg(dy + e), d);
    unpack8(__ldg(x + e), xv);
    if (relu) {
      const unsigned m = __ldg(mask + e);
#pragma unroll
      for (int i = 0; i < 8; ++i) d[i] = (m >> i) & 1u ? d[i] : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float xhat = (xv[i] - tab[c0 + i]) * tab[C + c0 + i];
      o[i] = tab[2 * C + c0 + i] * (d[i] - tab[3 * C + c0 + i] - xhat * tab[4 * C + c0 + i]);
    }
    dx[e] = pack8(o);
    if (dres != nullptr) dres[e] = pack8(d);
  }
}

// acc[col] = sum over p = 0..P-1 of part[p][col] (W = 2C columns), always in the same order: 32 columns per CTA,
// 32 warps each summing every 32nd row (few dependent loads per thread), then the 32 warp sums in warp order
constexpr int BN_SUM_THREADS = 1024;
__global__ void __launch_bounds__(BN_SUM_THREADS)
bn_sum_partials_kernel(const float* __restrict__ part, int P, int W, float* __restrict__ acc) {
  __shared__ float red[BN_SUM_THREADS / 32][32];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + lane;
  float s = 0.f;
  pdl_wait();
  if (col < W) {
#pragma unroll 4
    for (int p = g; p < P; p += BN_SUM_THREADS / 32) s += __ldg(part + (long long)p * W + col);
  }
  pdl_launch_dependents();
  red[g][lane] = s;
  __syncthreads();
  if (g == 0 && col < W) {
    float t = red[0][lane];
#pragma unroll
    for (int k = 1; k < BN_SUM_THREADS / 32; ++k) t += red[k][lane];
    acc[col] = t;
  }
}

// Launch with programmatic stream serialization: the grid may be scheduled while the previous kernel in the stream
// is still running, so the kernel must call pdl_wait() before its first global read or write.  A launch error is
// reported by cudaGetLastError(), as for a <<<>>> launch.
template <typename... Params, typename... Args>
static void launch_pdl(void (*kernel)(Params...), int grid, int block, size_t smem, cudaStream_t stream,
                       Args... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, args...);
}

extern "C" {

static int bn_grid(long long work_items, int per_block) {
  long long g = (work_items + per_block - 1) / per_block;
  if (g > num_sms() * 8) g = num_sms() * 8;
  if (g < 1) g = 1;
  return (int)g;
}
// reduction kernels: rows handled per thread, chosen so that even the small late layers (R = 2048)
// launch ~2 waves of CTAs instead of 32 latency-bound ones
static int g_bn_reduce_ctas = 0;
static int bn_reduce_grid(long long R, int RL) {
  // Every CTA ends with a 2C-float partial that bn_sum_partials_kernel reads back, so the grid is capped at a few
  // CTAs per SM (round 1 launched up to 1024 CTAs of one row per thread for the 2-4 MB layers, with global atomics:
  // slower than the 16 MB layers); the row loops keep 4-6 loads in flight per thread instead.
  if (g_bn_reduce_ctas == 0) {
    const char* e = getenv("ATOMO_BN_REDUCE_CTAS");
    g_bn_reduce_ctas = e != nullptr ? atoi(e) : 296;
    if (g_bn_reduce_ctas < 1) g_bn_reduce_ctas = 296;
  }
  long long g = (R + RL - 1) / RL;
  if (g > g_bn_reduce_ctas) g = g_bn_reduce_ctas;
  return (int)(g < 1 ? 1 : g);
}

// floats of the `part` scratch the launchers below need for a layer of R rows x C channels
long long atomo_bn_partial_floats(long long R, int C) {
  return (long long)bn_reduce_grid(R, BN_THREADS / (C / 8)) * 2 * C;
}

static void bn_sum_partials(const float* part, int P, int C, float* acc, cudaStream_t stream) {
  launch_pdl(bn_sum_partials_kernel, (2 * C + 31) / 32, BN_SUM_THREADS, 0, stream, part, P, 2 * C, acc);
}

// acc (2C floats) is overwritten with the layer's sums; part holds atomo_bn_partial_floats(R, C) floats.  With a mask
// (uint8 [R][C/8]) the output is ReLU'd and the mask receives its y > 0 bits.
void atomo_launch_bn_forward(const void* x, const void* res, void* y, void* mask, long long R, int C, float* acc,
                             float* part, const float* gamma, const float* beta, float* save_mean, float* save_invstd,
                             float* running_mean, float* running_var, float eps, float momentum, cudaStream_t stream) {
  const int CG = C / 8, RL = BN_THREADS / CG;
  const int g1 = bn_reduce_grid(R, RL);
  bn_stats_kernel<<<g1, BN_THREADS, 2 * RL * C * sizeof(float), stream>>>((const uint4*)x, R, C, part);
  bn_sum_partials(part, g1, C, acc, stream);
  const int g2 = bn_grid(R * CG, BN_THREADS * 2);
  launch_pdl(bn_apply_kernel, g2, BN_THREADS, 2 * C * sizeof(float), stream, (const uint4*)x, (const uint4*)res,
             (uint4*)y, (uint8_t*)mask, R, C, (const float*)acc, gamma, beta, save_mean, save_invstd, running_mean,
             running_var, eps, momentum, mask != nullptr ? 1 : 0);
}

// mask: the forward's ReLU mask, or nullptr for a layer without ReLU
void atomo_launch_bn_backward(const void* dy, const void* x, const void* mask, void* dx, void* dres, long long R, int C,
                              const float* mean, const float* invstd, const float* gamma, float* acc, float* part,
                              float* dgamma, float* dbeta, cudaStream_t stream) {
  const int CG = C / 8, RL = BN_THREADS / CG;
  const int relu = mask != nullptr ? 1 : 0;
  const int g1 = bn_reduce_grid(R, RL);
  bn_bwd_reduce_kernel<<<g1, BN_THREADS, 2 * RL * C * sizeof(float), stream>>>((const uint4*)dy, (const uint4*)x,
                                                                               (const uint8_t*)mask, R, C, mean,
                                                                               invstd, part, relu);
  bn_sum_partials(part, g1, C, acc, stream);
  const int g2 = bn_grid(R * CG, BN_THREADS * 2);
  launch_pdl(bn_bwd_apply_kernel, g2, BN_THREADS, 5 * C * sizeof(float), stream, (const uint4*)dy, (const uint4*)x,
             (const uint8_t*)mask, (uint4*)dx, (uint4*)dres, R, C, mean, invstd, gamma, (const float*)acc, dgamma,
             dbeta, relu);
}
}
}  // namespace atomo
