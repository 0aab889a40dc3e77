// Subspace-iteration route for square-ish layers (fc, 1x1 convolutions) — the part of K1 the
// reference does with a full LAPACK SVD of e.g. a 4096 x 9216 matrix on the host (svd.py:95).
//
//   Y = A X          (skinny GEMM, wgmma — gemm_kernels.cu)          m x l
//   Q = orth(Y)      (gram + eig_sample(top-l) + project on the aux plan: Q = Y V / sigma)
//   B = A^T Q        (skinny GEMM, wgmma)                            n x l
//   B = Ub S Vb^T    (gram + eig_sample(ATOMO sampling) + project on the aux plan)
//   A ~ (Q Vb) S Ub^T: this file's kernel forms U = Q Vb for the sampled atoms and stores
//   (U, S/p, Ub^T) straight into the PS slot over NVLink.
#include "common.cuh"

namespace atomo {

struct ExtDesc {
  long long a_off;       // gradient offset of the layer in the flat buffer
  long long xt_off;      // scratch: X^T (l x n)
  long long y_off;       // scratch: Y (m x l)
  long long b_off;       // scratch: B (n x l)
  long long qslot_off;   // local arena (aux_y): slot whose U part is Q (m x l)
  long long bslot_off;   // local arena (aux_b): slot {count, s, Vb (rcap x l), Ub (n x rcap)}
  long long ps_slot_off; // slot of this layer inside a worker arena on the PS
  long long pad0;
  int rows, cols, row_stride, col_stride;
  int sketch, rcap, layer, pad1;
};

constexpr int FIN_THREADS = 256;

__global__ void __launch_bounds__(FIN_THREADS)
ext_finalize_push_kernel(const ExtDesc* __restrict__ descs, const TileDesc* __restrict__ tiles,
                         const float* __restrict__ arena_y, const float* __restrict__ arena_b,
                         float* ps_arena_peer, long long arena_floats, const Ctrl* ctrl, int worker_index) {
  __shared__ __align__(16) float vb[RCAP_MAX * RCAP_MAX];  // Vb[a][j], a < rcap, j < l
  const TileDesc t = tiles[blockIdx.x];
  const ExtDesc D = descs[t.layer];
  const int l = D.sketch, rcap = D.rcap, n = D.cols;
  const float* bslot = arena_b + D.bslot_off;
  const int count = min(max(reinterpret_cast<const int*>(bslot)[0], 0), rcap);
  for (int e = threadIdx.x; e < rcap * l; e += blockDim.x) {
    const int a = e / l;
    vb[e] = (a < count) ? bslot[slot_v_off(rcap) + e] : 0.f;
  }
  __syncthreads();

  float* slot = ps_arena_peer + (long long)worker_index * arena_floats + D.ps_slot_off;
  // U[row][a] = sum_j Q[row][j] * Vb[a][j]
  const float* Q = arena_y + D.qslot_off + slot_u_off(l, l);
  float* U = slot + slot_u_off(rcap, n);
  const int c4 = (count + 3) >> 2;
  for (int r = threadIdx.x; r < t.nrows; r += blockDim.x) {
    const long long row = t.row0 + r;
    float q[RCAP_MAX];
    for (int j4 = 0; j4 < (l >> 2); ++j4) {
      const float4 v = *reinterpret_cast<const float4*>(Q + row * l + 4 * j4);
      q[4 * j4] = v.x; q[4 * j4 + 1] = v.y; q[4 * j4 + 2] = v.z; q[4 * j4 + 3] = v.w;
    }
    for (int g = 0; g < c4; ++g) {
      float o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int a = 4 * g + k;
        float acc = 0.f;
        if (a < count)
          for (int j = 0; j < l; ++j) acc = fmaf(q[j], vb[a * l + j], acc);
        o[k] = acc;
      }
      st_na_f4(reinterpret_cast<float4*>(U + row * rcap) + g, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
  // the first tile of each layer also publishes the header, s and V = Ub^T
  if (t.row0 == 0) {
    const float* Ub = bslot + slot_u_off(rcap, l);  // n x rcap
    for (int e = threadIdx.x; e < rcap * n; e += blockDim.x) {
      const int a = e / n, c = e - a * n;
      slot[slot_v_off(rcap) + e] = (a < count) ? Ub[(long long)c * rcap + a] : 0.f;
    }
    if (threadIdx.x < rcap) slot[slot_s_off() + threadIdx.x] = (threadIdx.x < count) ? bslot[slot_s_off() + threadIdx.x] : 0.f;
    if (threadIdx.x == 0) {
      int* hdr = reinterpret_cast<int*>(slot);
      hdr[0] = count; hdr[1] = ctrl->step; hdr[2] = n; hdr[3] = D.rows;
    }
  }
  __threadfence_system();
}

extern "C" {
void atomo_launch_ext_finalize(const void* descs, const void* tiles, int ntiles, const float* arena_y,
                               const float* arena_b, float* ps_arena_peer, long long arena_floats,
                               const void* ctrl, int worker_index, cudaStream_t stream) {
  if (ntiles <= 0) return;
  ext_finalize_push_kernel<<<ntiles, FIN_THREADS, 0, stream>>>((const ExtDesc*)descs, (const TileDesc*)tiles,
                                                                arena_y, arena_b, ps_arena_peer, arena_floats,
                                                                (const Ctrl*)ctrl, worker_index);
}
int atomo_ext_desc_bytes() { return (int)sizeof(ExtDesc); }
}
}  // namespace atomo
