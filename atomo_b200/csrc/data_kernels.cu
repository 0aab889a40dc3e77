// Training input built on the device: gather a batch of source images in the epoch's sample order, apply the
// CIFAR / SVHN augmentation (pad -> random crop -> random horizontal flip) and ToTensor + Normalize, and write the
// fp32 batch and its int64 labels.  One launch per batch, no host synchronisation (data/gpu_loader.py).
//
// Uint8 sources are NHWC.  Per sample, Philox keyed by (seed, epoch, position in the epoch) draws the crop offset
// (top, left) in [0, 2*pad] and the flip bit.  Reflect padding maps i < 0 to -i and i >= W to 2W-2-i (numpy's
// "reflect", which torchvision's TF.pad uses for PIL images); constant padding reads 0.  The value is
// (float(u8) / 255 - mean[c]) / std[c] with every operation an IEEE round-to-nearest intrinsic, so neither
// --use_fast_math nor FMA contraction can change it: it equals torchvision's fp32 to_tensor + normalize bit for bit.
// Fp32 sources (the synthetic datasets, NHWC) are gathered unchanged: their CPU pipeline has no augmentation.
#include "common.cuh"

namespace atomo {

constexpr int AUG_THREADS = 256;
constexpr uint32_t AUG_DOMAIN = 0x41554731u;  // Philox counter word separating these draws from the coders'

struct AugArgs {
  const void* src;            // [N, H, W, C] uint8 or fp32
  const long long* labels;    // [N]
  const int* order;           // the epoch's sample order (indices into src)
  const float* mean_std;      // [2, C]: mean then std, fp32
  const int* ext_draws;       // tests: [B, 3] (top, left, flip) replacing Philox, or nullptr
  float* x;                   // [B, C, H, W] at the strides below
  long long* y;               // [B]
  long long pos0;             // position of the batch's first sample in the epoch
  long long sx_n, sx_c, sx_h, sx_w;
  unsigned long long seed;
  int B, C, H, W;
  int pad, reflect, augment, src_u8;
  uint32_t epoch;
};

__device__ __forceinline__ int reflect_index(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// one thread per output pixel (all channels); the flat index runs over (sample, row, column)
__global__ void __launch_bounds__(AUG_THREADS) augment_gather_kernel(const AugArgs a) {
  const int hw = a.H * a.W;
  const long long idx = (long long)blockIdx.x * AUG_THREADS + threadIdx.x;
  if (idx >= (long long)a.B * hw) return;
  const int b = (int)(idx / hw);
  const int p = (int)(idx - (long long)b * hw);
  const int h = p / a.W, w = p - h * a.W;
  const long long pos = a.pos0 + b;
  const long long s = a.order[pos];

  int top = a.pad, left = a.pad, flip = 0;
  if (a.augment) {
    if (a.ext_draws != nullptr) {
      top = a.ext_draws[3 * b];
      left = a.ext_draws[3 * b + 1];
      flip = a.ext_draws[3 * b + 2] & 1;
    } else {
      uint32_t r[4];
      Philox::gen(a.seed, (uint32_t)pos, (uint32_t)(pos >> 32), a.epoch, AUG_DOMAIN, r);
      const uint64_t span = 2 * a.pad + 1;
      top = (int)(((uint64_t)r[0] * span) >> 32);
      left = (int)(((uint64_t)r[1] * span) >> 32);
      flip = r[2] >> 31;
    }
  }
  int sr = h + top - a.pad;
  int sc = (flip ? a.W - 1 - w : w) + left - a.pad;
  float* out = a.x + b * a.sx_n + h * a.sx_h + w * a.sx_w;
  if (a.src_u8) {
    bool inside = true;
    if (a.reflect) {
      sr = reflect_index(sr, a.H);
      sc = reflect_index(sc, a.W);
    } else {
      inside = sr >= 0 && sr < a.H && sc >= 0 && sc < a.W;
    }
    const unsigned char* px = (const unsigned char*)a.src + ((s * a.H + (inside ? sr : 0)) * a.W + (inside ? sc : 0)) * a.C;
    for (int c = 0; c < a.C; ++c) {
      const float u = inside ? (float)px[c] : 0.0f;
      const float t = __fsub_rn(__fdiv_rn(u, 255.0f), a.mean_std[c]);
      out[c * a.sx_c] = __fdiv_rn(t, a.mean_std[a.C + c]);
    }
  } else {
    const float* px = (const float*)a.src + ((s * a.H + sr) * a.W + sc) * a.C;
    for (int c = 0; c < a.C; ++c) out[c * a.sx_c] = px[c];
  }
  if (p == 0) a.y[b] = a.labels[s];
}

extern "C" {

void atomo_launch_augment_gather(const void* src, int src_u8, const long long* labels, int C, int H, int W,
                                 const int* order, long long pos0, int B, const float* mean_std, int pad, int reflect,
                                 int augment, unsigned long long seed, int epoch, const int* ext_draws, float* x,
                                 long long sx_n, long long sx_c, long long sx_h, long long sx_w, long long* y,
                                 cudaStream_t stream) {
  AugArgs a;
  a.src = src; a.labels = labels; a.order = order; a.mean_std = mean_std; a.ext_draws = ext_draws;
  a.x = x; a.y = y; a.pos0 = pos0;
  a.sx_n = sx_n; a.sx_c = sx_c; a.sx_h = sx_h; a.sx_w = sx_w;
  a.seed = seed; a.B = B; a.C = C; a.H = H; a.W = W;
  a.pad = pad; a.reflect = reflect; a.augment = augment; a.src_u8 = src_u8; a.epoch = (uint32_t)epoch;
  const long long n = (long long)B * H * W;
  const long long grid = (n + AUG_THREADS - 1) / AUG_THREADS;
  if (grid < 1) return;
  augment_gather_kernel<<<(unsigned)grid, AUG_THREADS, 0, stream>>>(a);
}

}  // extern "C"
}  // namespace atomo
