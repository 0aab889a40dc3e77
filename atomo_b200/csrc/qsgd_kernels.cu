// K5/K6 — QSGD / TernGrad quantize + bit-pack fused with the worker->PS push,
// and the PS-side unpack + aggregate (sm_90a).
//
// Reference (SURVEY.md 2.5 K5/K6): numpy encode with a Python loop over the
// floor(64/(2+q)) sections (codings/qsgd.py:19-87), or ~15 separate torch CUDA
// launches (qsgd.py:157-209); numpy Python-loop decode (qsgd.py:89-151).
// Here: ONE pass.  A warp owns one bucket (default 512 elements): coalesced load,
// warp-shuffle L2 / L-inf norm, Philox stochastic rounding (unbiased: round up
// with probability frac — the reference's inverted rule is not replicated),
// (sign+1)<<q | level codes staged in shared memory, section-major 64-bit word
// assembly, and the words + bucket norms are stored straight into the PS arena
// through NVLink peer pointers.  Wire layout == atomo_b200.codings.qsgd.
#include "common.cuh"

namespace atomo {

constexpr int Q_WARPS = 8;
constexpr int Q_MAX_BUCKET = 1024;

__device__ __forceinline__ int q_words_per_bucket(int bucket, int q) {
  const int E = 64 / (2 + q);
  return (bucket + E - 1) / E;
}

__global__ void __launch_bounds__(Q_WARPS * 32)
qsgd_encode_kernel(const float* __restrict__ grad, long long numel, int bucket, int q, int terngrad,
                   const float* __restrict__ clip_ptr, unsigned long long* words_out, float* norms_out,
                   const Ctrl* ctrl, int worker_index, const float* __restrict__ ext_uniforms, long long nbuckets) {
  __shared__ unsigned short codes[Q_WARPS][Q_MAX_BUCKET];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int levels = (1 << q) - 1;
  const int E = 64 / (2 + q);
  const int L = q_words_per_bucket(bucket, q);
  const float clip = (terngrad && clip_ptr != nullptr) ? *clip_ptr : 0.f;
  const int step = ctrl->step;

  for (long long b = (long long)blockIdx.x * Q_WARPS + warp; b < nbuckets; b += (long long)gridDim.x * Q_WARPS) {
    const long long base = b * bucket;
    // pass 1: norm
    float nrm = 0.f;
    for (int i = lane; i < bucket; i += 32) {
      const long long e = base + i;
      float x = e < numel ? __ldg(grad + e) : 0.f;
      if (terngrad) {
        if (clip > 0.f) x = fminf(fmaxf(x, -clip), clip);
        nrm = fmaxf(nrm, fabsf(x));
      } else {
        nrm = fmaf(x, x, nrm);
      }
    }
    nrm = terngrad ? warp_max(nrm) : sqrtf(warp_sum(nrm));
    const float inv = nrm > 0.f ? (float)levels / nrm : 0.f;
    // pass 2: stochastic quantization -> codes (the bucket is L1/L2 resident from pass 1)
    for (int i = lane; i < bucket; i += 32) {
      const long long e = base + i;
      float x = e < numel ? __ldg(grad + e) : 0.f;
      if (terngrad && clip > 0.f) x = fminf(fmaxf(x, -clip), clip);
      const float a = fminf(fabsf(x) * inv, (float)levels);
      const float lo = floorf(a);
      const float frac = a - lo;
      float u;
      if (ext_uniforms != nullptr) {
        u = ext_uniforms[e < numel ? e : 0];
      } else {
        uint32_t r4[4];
        Philox::gen(ctrl->seed ^ 0x5151515151515151ULL, (uint32_t)e, (uint32_t)(e >> 32), (uint32_t)step,
                    (uint32_t)worker_index, r4);
        u = Philox::to_uniform(r4[0]);
      }
      int xi = (int)lo + (u < frac ? 1 : 0);
      xi = min(xi, levels);
      const int sgn = (x > 0.f) ? 2 : (x < 0.f ? 0 : 1);
      codes[warp][i] = (unsigned short)((sgn << q) | xi);
    }
    __syncwarp();
    // section-major packing: word j holds elements j, j+L, j+2L, ... (section 0 in the MSBs)
    for (int j = lane; j < L; j += 32) {
      unsigned long long w = 0ULL;
      for (int s = 0; s < E; ++s) {
        const int i = s * L + j;
        const unsigned long long c = (i < bucket) ? (unsigned long long)codes[warp][i] : (1ULL << q);
        w = (w << (2 + q)) | c;
      }
      words_out[b * L + j] = w;
    }
    if (lane == 0) norms_out[b] = nrm;
    __syncwarp();
  }
}

// PS side: out_sum[e] = sum_w decode_w[e]   (terngrad: every worker's code is scaled by the max norm,
// qsgd.py:103-104 / 153-155).  Waits for the workers' push flags first when given.
__global__ void __launch_bounds__(Q_WARPS * 32)
qsgd_decode_sum_kernel(const unsigned long long* const* words, const float* const* norms, int W, long long numel,
                       int bucket, int q, int terngrad, float* __restrict__ out_sum, long long nbuckets,
                       const int* push_flags, Ctrl* ctrl, long long timeout_ticks) {
  __shared__ unsigned long long wsm[Q_WARPS][Q_MAX_BUCKET / 2];
  __shared__ int s_ok;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (push_flags != nullptr) {
    if (threadIdx.x == 0) {
      bool ok = true;
      for (int w = 0; w < W; ++w) ok = spin_wait_ge(push_flags + w, ctrl->step, timeout_ticks) && ok;
      if (!ok) atomicExch(&ctrl->error, ERR_WAIT_PUSH_TIMEOUT);
      s_ok = ok;
    }
    __syncthreads();
    if (!s_ok) return;
  }
  const int levels = (1 << q) - 1;
  const int E = 64 / (2 + q);
  const int L = q_words_per_bucket(bucket, q);
  const unsigned long long mask = (1ULL << (2 + q)) - 1ULL;
  const float inv_levels = 1.f / (float)levels;

  for (long long b = (long long)blockIdx.x * Q_WARPS + warp; b < nbuckets; b += (long long)gridDim.x * Q_WARPS) {
    float nmax = 0.f;
    if (terngrad)
      for (int w = 0; w < W; ++w) nmax = fmaxf(nmax, ld_cg_f(norms[w] + b));
    float acc[Q_MAX_BUCKET / 32];
#pragma unroll
    for (int t = 0; t < Q_MAX_BUCKET / 32; ++t) acc[t] = 0.f;
    for (int w = 0; w < W; ++w) {
      const float scale = (terngrad ? nmax : ld_cg_f(norms[w] + b)) * inv_levels;
      __syncwarp();
      for (int j = lane; j < L; j += 32) {
        unsigned long long v;
        asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(v) : "l"(words[w] + b * L + j));
        wsm[warp][j] = v;
      }
      __syncwarp();
#pragma unroll
      for (int t = 0; t < Q_MAX_BUCKET / 32; ++t) {
        const int i = lane + 32 * t;
        if (i < bucket) {
          const int s = i / L, j = i - s * L;
          const unsigned long long c = (wsm[warp][j] >> ((E - 1 - s) * (2 + q))) & mask;
          const float xi = (float)(c & (unsigned long long)levels);
          const float sg = (float)((int)(c >> q) & 3) - 1.f;
          acc[t] = fmaf(sg * xi, scale, acc[t]);
        }
      }
    }
    const long long base = b * bucket;
#pragma unroll
    for (int t = 0; t < Q_MAX_BUCKET / 32; ++t) {
      const int i = lane + 32 * t;
      if (i < bucket && base + i < numel) out_sum[base + i] = acc[t];
    }
  }
}

extern "C" {

void atomo_launch_qsgd_encode(const float* grad, long long numel, int bucket, int q, int terngrad,
                              const float* clip_ptr, unsigned long long* words_out, float* norms_out,
                              const void* ctrl, int worker_index, const float* ext_uniforms, cudaStream_t stream) {
  const long long nb = (numel + bucket - 1) / bucket;
  long long grid = (nb + Q_WARPS - 1) / Q_WARPS;
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  if (grid < 1) grid = 1;
  qsgd_encode_kernel<<<(int)grid, Q_WARPS * 32, 0, stream>>>(grad, numel, bucket, q, terngrad, clip_ptr, words_out,
                                                              norms_out, (const Ctrl*)ctrl, worker_index,
                                                              ext_uniforms, nb);
}

void atomo_launch_qsgd_decode_sum(const unsigned long long* const* words, const float* const* norms, int W,
                                  long long numel, int bucket, int q, int terngrad, float* out_sum,
                                  const int* push_flags, void* ctrl, long long timeout_ticks, cudaStream_t stream) {
  const long long nb = (numel + bucket - 1) / bucket;
  long long grid = (nb + Q_WARPS - 1) / Q_WARPS;
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  if (grid < 1) grid = 1;
  qsgd_decode_sum_kernel<<<(int)grid, Q_WARPS * 32, 0, stream>>>(words, norms, W, numel, bucket, q, terngrad,
                                                                  out_sum, nb, push_flags, (Ctrl*)ctrl,
                                                                  timeout_ticks);
}

int atomo_qsgd_max_bucket() { return Q_MAX_BUCKET; }

}  // extern "C"
}  // namespace atomo
