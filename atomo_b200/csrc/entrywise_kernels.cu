// K3/K4 — entry-wise ATOMO (standard-basis atoms) fused with the worker->PS push,
// and the PS-side scatter-add (sm_90a).
//
// Reference: the scheme is the ATOMO recipe applied to the standard basis
// (README.md:5-7; only the L1 indicator exists in code, codings/utils.py:7-8).
// p_i = min(1, s_l * |g_i| / ||g_l||_1) with s_l = budget * numel_l per tensor l;
// element i is kept with probability p_i and sent as (flat index, g_i / p_i).
//
//   l1_kernel        : per-tensor L1 norms (grouped over the dense tile table)
//   sample_push      : Philox Bernoulli sampling, warp-ballot compaction with one
//                      warp-aggregated atomic per warp, (idx,val) pairs stored
//                      straight into the PS arena through NVLink peer pointers;
//                      the last CTA publishes the count and the step flag
//   scatter_kernel   : PS side: atomicAdd of every worker's list into a dense
//                      fp32 sum buffer (then the fused SGD+broadcast kernel runs).
#include "common.cuh"

namespace atomo {

constexpr int EW_THREADS = 256;

__global__ void __launch_bounds__(EW_THREADS)
entrywise_l1_kernel(const float* __restrict__ grad, const LayerDesc* __restrict__ layers,
                    const TileDesc* __restrict__ tiles, int ntiles, float* __restrict__ l1) {
  __shared__ float part[EW_THREADS / 32];
  for (int ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
    const TileDesc t = tiles[ti];
    const LayerDesc L = layers[t.layer];
    const float* base = grad + L.off + (long long)t.row0 * 4;
    float s = 0.f;
    for (int i = threadIdx.x; i < t.nrows; i += blockDim.x) s += fabsf(__ldg(base + i));
    s = warp_sum(s);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int w = 0; w < EW_THREADS / 32; ++w) tot += part[w];
      atomicAdd(l1 + t.layer, tot);
    }
  }
}

__global__ void __launch_bounds__(EW_THREADS)
entrywise_sample_push_kernel(const float* __restrict__ grad, const LayerDesc* __restrict__ layers,
                             const TileDesc* __restrict__ tiles, int ntiles, const float* __restrict__ l1,
                             float budget, int* idx_out, float* val_out, int* count_out, int capacity,
                             int* local_count, int* push_flag_peer, Ctrl* ctrl, int worker_index,
                             const float* __restrict__ ext_uniforms, int signal) {
  const int lane = threadIdx.x & 31;
  const int step = ctrl->step;
  for (int ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
    const TileDesc t = tiles[ti];
    const LayerDesc L = layers[t.layer];
    const long long e0 = L.off + (long long)t.row0 * 4;
    const float norm = l1[t.layer];
    // budget < 1: fraction of the tensor; budget >= 1: absolute expected atom count
    float s = budget < 1.f ? budget * (float)L.numel : budget;
    s = fminf(fmaxf(s, 1.f), (float)L.numel);
    const float scale = norm > 0.f ? s / norm : 0.f;
    const int iters = (t.nrows + blockDim.x - 1) / blockDim.x;
    for (int it = 0; it < iters; ++it) {
      const int i = it * blockDim.x + threadIdx.x;
      bool keep = false;
      float val = 0.f;
      long long e = e0 + i;
      if (i < t.nrows) {
        const float g = __ldg(grad + e);
        const float p = fminf(fabsf(g) * scale, 1.f);
        float u;
        if (ext_uniforms != nullptr) {
          u = ext_uniforms[e];
        } else {
          uint32_t r4[4];
          Philox::gen(ctrl->seed ^ 0xE17E17E17E17E17EULL, (uint32_t)e, (uint32_t)(e >> 32), (uint32_t)step,
                      (uint32_t)worker_index, r4);
          u = Philox::to_uniform(r4[0]);
        }
        keep = u < p;
        val = keep ? g / p : 0.f;
      }
      const unsigned int m = __ballot_sync(0xffffffffu, keep);
      if (m) {
        int basepos = 0;
        if (lane == 0) basepos = atomicAdd(local_count, __popc(m));
        basepos = __shfl_sync(0xffffffffu, basepos, 0);
        if (keep) {
          const int pos = basepos + __popc(m & ((1u << lane) - 1u));
          if (pos < capacity) {
            idx_out[pos] = (int)e;
            val_out[pos] = val;
          } else {
            atomicExch(&ctrl->error, ERR_SLOT_OVERFLOW);
          }
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned int old = atomicAdd(&ctrl->done_aux, 1u);
    if (old == gridDim.x - 1) {
      ctrl->done_aux = 0;
      const int c = min(*local_count, capacity);
      *local_count = 0;
      *count_out = c;
      __threadfence_system();
      if (signal) st_release_sys(push_flag_peer + worker_index, step);
    }
  }
}

// PS: out_sum[idx] += val for every (idx,val) of every worker
__global__ void __launch_bounds__(EW_THREADS)
entrywise_scatter_kernel(const int* const* idx, const float* const* val, const int* const* count, int W,
                         int capacity, float* __restrict__ out_sum, long long numel, const int* push_flags,
                         Ctrl* ctrl, long long timeout_ticks) {
  __shared__ int s_ok;
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
  for (int w = 0; w < W; ++w) {
    const int n = min(ld_cg_i(count[w]), capacity);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
      const int e = ld_cg_i(idx[w] + i);
      if (e >= 0 && e < numel) atomicAdd(out_sum + e, ld_cg_f(val[w] + i));
    }
  }
}

extern "C" {

void atomo_launch_entrywise_encode(const float* grad, const void* layers, const void* tiles, int ntiles, float* l1,
                                   int nlayers, float budget, int* idx_out, float* val_out, int* count_out,
                                   int capacity, int* local_count, int* push_flag_peer, void* ctrl,
                                   int worker_index, const float* ext_uniforms, int signal, cudaStream_t stream) {
  cudaMemsetAsync(l1, 0, sizeof(float) * nlayers, stream);
  int grid = ntiles < num_sms() * 4 ? ntiles : num_sms() * 4;
  if (grid < 1) grid = 1;
  entrywise_l1_kernel<<<grid, EW_THREADS, 0, stream>>>(grad, (const LayerDesc*)layers, (const TileDesc*)tiles,
                                                        ntiles, l1);
  entrywise_sample_push_kernel<<<grid, EW_THREADS, 0, stream>>>(
      grad, (const LayerDesc*)layers, (const TileDesc*)tiles, ntiles, l1, budget, idx_out, val_out, count_out,
      capacity, local_count, push_flag_peer, (Ctrl*)ctrl, worker_index, ext_uniforms, signal);
}

void atomo_launch_entrywise_scatter(const int* const* idx, const float* const* val, const int* const* count, int W,
                                    int capacity, float* out_sum, long long numel, const int* push_flags,
                                    void* ctrl, long long timeout_ticks, cudaStream_t stream) {
  cudaMemsetAsync(out_sum, 0, sizeof(float) * numel, stream);
  int grid = (capacity + EW_THREADS - 1) / EW_THREADS;
  if (grid > num_sms() * 4) grid = num_sms() * 4;
  if (grid < 1) grid = 1;
  entrywise_scatter_kernel<<<grid, EW_THREADS, 0, stream>>>(idx, val, count, W, capacity, out_sum, numel,
                                                             push_flags, (Ctrl*)ctrl, timeout_ticks);
}

}  // extern "C"
}  // namespace atomo
