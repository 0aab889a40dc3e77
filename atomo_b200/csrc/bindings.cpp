// Python bindings for the atomo_b200 native runtime (torch extension `atomo_b200._C`).
// Kernels live in the .cu files behind a plain C ABI; this file only adapts
// torch tensors / raw peer pointers to those launchers on the current stream.
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAEvent.h>
#include <c10/cuda/CUDACachingAllocator.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cstdint>
#include <string>

extern "C" {
// symm_heap.cpp
const char* atomo_heap_last_error();
int atomo_heap_multicast_supported(int device);
int atomo_heap_posix_fd_supported(int device);
void* atomo_heap_create_vmm(int rank, int world, int device, size_t bytes, const char* job, int want_mc,
                            double timeout_s);
int atomo_heap_mc_phase_a(void* h, double timeout_s);
int atomo_heap_mc_phase_b(void* h);
void* atomo_heap_create_ipc(int rank, int world, int device, size_t bytes, unsigned char* handle_out64);
int atomo_heap_open_ipc(void* h, const unsigned char* all_handles);
uint64_t atomo_heap_ptr(void* h, int rank);
uint64_t atomo_heap_mc_ptr(void* h);
uint64_t atomo_heap_bytes(void* h);
const char* atomo_heap_mode(void* h);
void atomo_heap_destroy(void* h);
// svd_kernels.cu
void atomo_launch_gram(const float* grad, const void* layers, const void* tiles, int ntiles, float* gpart,
                       cudaStream_t stream);
void atomo_launch_eig_sample(const void* layers, const int* ts_layers, int n_ts, const float* gpart, float* vsel,
                             int* selcount, float* sigma_out, float* ps_arena_peer, long long arena_floats,
                             const void* ctrl, const float* ext_uniforms, int rank, int random_sample,
                             int waterfill, int systematic, int worker_index, int threads, cudaStream_t stream);
void atomo_launch_project_push(const float* grad, const void* layers, const void* tiles, int ntiles,
                               const float* vsel, const int* selcount, float* ps_arena_peer,
                               long long arena_floats, int* push_flag_peer, void* ctrl, int worker_index,
                               int signal, cudaStream_t stream);
void atomo_launch_signal_push(int* push_flag_peer, const void* ctrl, int worker_index, cudaStream_t stream);
// ps_kernels.cu
int atomo_ps_smem_bytes();
int atomo_ps_tile_elems();
int atomo_ps_max_rows();
int atomo_ps_dense_elems();
int atomo_ps_max_workers();
void atomo_launch_ps_update(const void* layers, const void* tiles, int ntiles, int W, int nflags, int nranks,
                            float* params, float* momentum, float* const* params_peer, float* params_mc,
                            const float* const* grads_peer, const float* grads_mc, const float* arenas,
                            long long arena_floats, int* push_flags, int* const* param_flag_peer, void* ctrl,
                            long long timeout_ticks, float inv_w, int grid, long long* tstats, cudaStream_t stream);
void atomo_launch_wait_params(const int* param_flag, void* ctrl, long long timeout_ticks, long long* tstats,
                              cudaStream_t stream);
void atomo_launch_advance_step(void* ctrl, cudaStream_t stream);
void atomo_launch_param_bcast(const float* src, float* const* params_peer, float* params_mc, int nranks,
                              int self_rank, long long numel, cudaStream_t stream);
void atomo_launch_set_flags(int* const* flag_peer, int nranks, int value, cudaStream_t stream);
// bn_kernels.cu
long long atomo_bn_partial_floats(long long R, int C);
void atomo_launch_bn_forward(const void* x, const void* res, void* y, void* mask, long long R, int C, float* acc,
                             float* part, const float* gamma, const float* beta, float* save_mean, float* save_invstd,
                             float* running_mean, float* running_var, float eps, float momentum, cudaStream_t stream);
void atomo_launch_bn_backward(const void* dy, const void* x, const void* mask, void* dx, void* dres, long long R, int C,
                              const float* mean, const float* invstd, const float* gamma, float* acc, float* part,
                              float* dgamma, float* dbeta, cudaStream_t stream);
// v2_encode.cu / v2_ps.cu (overlapped, sharded bf16 engine)
int atomo_v2_unit_bytes();
int atomo_v2_ctrl_bytes();
int atomo_v2_enc_smem();
int atomo_v2_ps_smem();
int atomo_v2_ps_tile_elems();
void atomo_v2_launch_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                            float* gpart, unsigned int* unit_counters, float* vsel, int* selcount, float* sigma_out,
                            float* const* arena_peer, int n_owners, long long arena_floats, void* stage,
                            const void* ctrl, const float* ext_uniforms, float* vprev, int max_sweeps,
                            int random_sample, int waterfill, int systematic, int worker, int resample_empty,
                            int flags, long long* tstats, int group, cudaStream_t stream);
void atomo_v2_launch_project(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                             const float* vsel, const int* selcount, float* const* arena_peer, int* const* sig_peer,
                             int n_owners, long long arena_floats, int worker, int group, void* ctrl,
                             unsigned int* group_counter, int flags, long long* tstats, int final_group, int timed,
                             float* residual, int ef_owner, cudaStream_t stream);
void atomo_v2_launch_ps(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                        int final_group, int owner, float* master, float* mom, float* sq, float* sqmax, float* vmom,
                        float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer, float* vparams_local,
                        float* vparams_mc, float* const* vparams_peer, const float* vgrads_mc,
                        const float* const* vgrads_peer, const void* const* stage_peer, const float* arenas,
                        long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                        unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                        cudaStream_t stream);
void atomo_v2_launch_wait_params(const int* sig, int n_owners, void* ctrl, long long timeout, long long* tstats,
                                 cudaStream_t stream);
// v2_qsgd.cu (QSGD / TernGrad units of the bf16 engine)
void atomo_v2_launch_qsgd_stats(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                double* partials, unsigned int* unit_counters, float* clip, long long* tstats,
                                int group, cudaStream_t stream);
void atomo_v2_launch_qsgd_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 const float* clip, float* const* arena_peer, int* const* sig_peer, int n_owners,
                                 long long arena_floats, int worker, int group, const void* ctrl,
                                 unsigned int* group_counter, const float* ext_uniforms, long long* tstats,
                                 int final_group, int stamp_start, float* residual, cudaStream_t stream);
void atomo_v2_launch_ps_qsgd(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                             int final_group, int owner, float* master, float* mom, float* sq, float* sqmax,
                             float* vmom, float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer,
                             float* vparams_local, float* vparams_mc, float* const* vparams_peer,
                             const float* vgrads_mc, const float* const* vgrads_peer, const float* arenas,
                             long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                             unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                             cudaStream_t stream);
// v2_entrywise.cu (entry-wise ATOMO units of the bf16 engine)
void atomo_v2_launch_entry_stats(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 double* partials, unsigned int* unit_counters, double* l1, long long* tstats,
                                 int group, cudaStream_t stream);
void atomo_v2_launch_entry_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                  const double* l1, float* const* arena_peer, int* const* sig_peer, int n_owners,
                                  long long arena_floats, int worker, int group, const void* ctrl,
                                  unsigned int* group_counter, const float* ext_uniforms, long long* tstats,
                                  int final_group, float* residual, cudaStream_t stream);
void atomo_v2_launch_ps_entry(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks,
                              int group, int final_group, int owner, float* master, float* mom, float* sq,
                              float* sqmax, float* vmom, float* vsq, float* vsqmax, void* wshadow_mc,
                              void* const* wshadow_peer, float* vparams_local, float* vparams_mc,
                              float* const* vparams_peer, const float* vgrads_mc, const float* const* vgrads_peer,
                              const float* arenas, long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                              unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                              cudaStream_t stream);
// v2_topk.cu (top-k units of the bf16 engine; the PS is v2_ps_entry)
int atomo_v2_topk_state_ints();
int atomo_v2_topk_hist_bins();
int atomo_v2_topk_tile_bins();
void atomo_v2_launch_topk_select(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 int* hist, int* tile_counts, unsigned int* unit_counters, int* sel, long long* tstats,
                                 int group, cudaStream_t stream);
void atomo_v2_launch_topk_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 const int* sel, const int* tile_counts, float* const* arena_peer,
                                 int* const* sig_peer, int n_owners, long long arena_floats, int worker, int group,
                                 const void* ctrl, unsigned int* group_counter, long long* tstats, int final_group,
                                 float* residual, cudaStream_t stream);
void atomo_v2_launch_topk_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                     const long long* gptr, const int* sel, const int* tile_counts,
                                     float* const* arena_peer, int n_owners, long long arena_floats, int worker,
                                     double* partials, unsigned int* unit_counters, double* acc, cudaStream_t stream);
// v2_sign.cu (scaled-sign units of the bf16 engine)
void atomo_v2_launch_sign_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                 float* const* arena_peer, int* const* sig_peer, int n_owners, long long arena_floats,
                                 int worker, int group, const void* ctrl, unsigned int* group_counter,
                                 long long* tstats, int final_group, float* residual, cudaStream_t stream);
void atomo_v2_launch_ps_sign(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                             int final_group, int owner, float* master, float* mom, float* sq, float* sqmax,
                             float* vmom, float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer,
                             float* vparams_local, float* vparams_mc, float* const* vparams_peer,
                             const float* vgrads_mc, const float* const* vgrads_peer, const float* arenas,
                             long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                             unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                             cudaStream_t stream);
void atomo_v2_launch_sign_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                     const long long* gptr, float* const* arena_peer, int n_owners,
                                     long long arena_floats, int worker, double* partials, unsigned int* unit_counters,
                                     double* acc, cudaStream_t stream);
// v2_fp8.cu (fp8 units of the bf16 engine)
void atomo_v2_launch_fp8_encode(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                float* const* arena_peer, int* const* sig_peer, int n_owners, long long arena_floats,
                                int worker, int group, const void* ctrl, unsigned int* group_counter,
                                long long* tstats, int final_group, float* residual, cudaStream_t stream);
void atomo_v2_launch_ps_fp8(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks, int group,
                            int final_group, int owner, float* master, float* mom, float* sq, float* sqmax,
                            float* vmom, float* vsq, float* vsqmax, void* wshadow_mc, void* const* wshadow_peer,
                            float* vparams_local, float* vparams_mc, float* const* vparams_peer,
                            const float* vgrads_mc, const float* const* vgrads_peer, const float* arenas,
                            long long arena_floats, int* sig, int* const* sig_peer, void* ctrl,
                            unsigned int* group_counter, long long timeout, long long* tstats, float inv_w, int grid,
                            cudaStream_t stream);
void atomo_v2_launch_fp8_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                    const long long* gptr, float* const* arena_peer, int n_owners,
                                    long long arena_floats, int worker, double* partials, unsigned int* unit_counters,
                                    double* acc, cudaStream_t stream);
// v2_powersgd.cu (PowerSGD units of the bf16 engine)
int atomo_v2_powersgd_state_bytes();
void atomo_v2_launch_powersgd_init(const void* units, int n_units, float* scratch, const void* ctrl,
                                   cudaStream_t stream);
void atomo_v2_launch_powersgd_encode(const void* units, const void* enc_tiles, int tile0, int ntiles,
                                     const void* pw_tiles, int pw0, int npw, const long long* gptr, float* scratch,
                                     double* gram, void* state, void* stage, float* const* arena_peer,
                                     int* const* sig_peer, int n_owners, long long arena_floats, int worker, int group,
                                     const void* ctrl, unsigned int* group_counter, long long* tstats,
                                     int final_group, float* residual, cudaStream_t stream);
void atomo_v2_launch_ps_powersgd(const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks,
                                 int group, int final_group, int owner, float* master, float* mom, float* sq,
                                 float* sqmax, float* vmom, float* vsq, float* vsqmax, void* wshadow_mc,
                                 void* const* wshadow_peer, float* vparams_local, float* vparams_mc,
                                 float* const* vparams_peer, const float* vgrads_mc, const float* const* vgrads_peer,
                                 const void* const* stage_peer, const float* arenas, long long arena_floats, int* sig,
                                 int* const* sig_peer, void* ctrl, unsigned int* group_counter, long long timeout,
                                 long long* tstats, float inv_w, int grid, cudaStream_t stream);
void atomo_v2_launch_powersgd_code_stats(const void* units, const void* tiles, int tile0, int ntiles,
                                         const long long* gptr, float* scratch, const void* state, double* partials,
                                         unsigned int* unit_counters, double* acc, cudaStream_t stream);
// v2_feedback.cu (error feedback of the bf16 engine)
int atomo_v2_ef_chunk_bytes();
void atomo_v2_launch_ef_apply(const void* chunks, int chunk0, int nchunks, const long long* gptr, float* residual,
                              cudaStream_t stream);
// v2_stats.cu (estimator statistics of the bf16 engine, --code-stats)
int atomo_v2_stats_fields();
int atomo_v2_stats_partials();
void atomo_v2_launch_code_stats(const void* units, const void* tiles, int tile0, int ntiles, const long long* gptr,
                                const float* sigma, const int* selcount, const double* l1, const float* clip,
                                float* const* arena_peer, int n_owners, long long arena_floats, int worker,
                                int random_sample, int waterfill, double* partials, unsigned int* unit_counters,
                                double* acc, cudaStream_t stream);
void atomo_v2_launch_advance_step(void* ctrl, cudaStream_t stream);
void atomo_v2_launch_bcast_bytes(const void* src, void* const* peer, void* mc, int nranks, int self, long long nbytes,
                                 cudaStream_t stream);
// gemm_kernels.cu
int atomo_gemm_tile_bytes();
int atomo_gemm_smem_bytes();
void atomo_launch_skinny_gemm(const void* tiles, int ntiles, void* ctrl, int grid, cudaStream_t stream);
// ext_kernels.cu
void atomo_launch_ext_finalize(const void* descs, const void* tiles, int ntiles, const float* arena_y,
                               const float* arena_b, float* ps_arena_peer, long long arena_floats,
                               const void* ctrl, int worker_index, cudaStream_t stream);
int atomo_ext_desc_bytes();
// qsgd_kernels.cu / entrywise_kernels.cu
void atomo_launch_qsgd_encode(const float* grad, long long numel, int bucket, int q, int terngrad,
                              const float* clip_ptr, unsigned long long* words_out, float* norms_out,
                              const void* ctrl, int worker_index, const float* ext_uniforms, cudaStream_t stream);
void atomo_launch_qsgd_decode_sum(const unsigned long long* const* words, const float* const* norms, int W,
                                  long long numel, int bucket, int q, int terngrad, float* out_sum,
                                  const int* push_flags, void* ctrl, long long timeout_ticks, cudaStream_t stream);
int atomo_qsgd_max_bucket();
void atomo_launch_entrywise_encode(const float* grad, const void* layers, const void* tiles, int ntiles, float* l1,
                                   int nlayers, float budget, int* idx_out, float* val_out, int* count_out,
                                   int capacity, int* local_count, int* push_flag_peer, void* ctrl,
                                   int worker_index, const float* ext_uniforms, int signal, cudaStream_t stream);
void atomo_launch_entrywise_scatter(const int* const* idx, const float* const* val, const int* const* count, int W,
                                    int capacity, float* out_sum, long long numel, const int* push_flags,
                                    void* ctrl, long long timeout_ticks, cudaStream_t stream);
// data_kernels.cu
void atomo_launch_augment_gather(const void* src, int src_u8, const long long* labels, int C, int H, int W,
                                 const int* order, long long pos0, int B, const float* mean_std, int pad, int reflect,
                                 int augment, unsigned long long seed, int epoch, const int* ext_draws, float* x,
                                 long long sx_n, long long sx_c, long long sx_h, long long sx_w, long long* y,
                                 cudaStream_t stream);
}

namespace {

inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
template <typename T>
inline T* P(uint64_t v) { return reinterpret_cast<T*>(static_cast<uintptr_t>(v)); }

void check_cuda_f32(const torch::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.scalar_type() == torch::kFloat32, name, " must be float32");
  TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}

// ---------------------------------------------------------------------------------------------- heap
uint64_t heap_create_vmm(int rank, int world, int device, uint64_t bytes, const std::string& job, bool want_mc,
                         double timeout_s) {
  void* h = atomo_heap_create_vmm(rank, world, device, bytes, job.c_str(), want_mc ? 1 : 0, timeout_s);
  return reinterpret_cast<uint64_t>(h);
}
py::tuple heap_create_ipc(int rank, int world, int device, uint64_t bytes) {
  unsigned char handle[64] = {0};
  void* h = atomo_heap_create_ipc(rank, world, device, bytes, handle);
  return py::make_tuple(reinterpret_cast<uint64_t>(h), py::bytes(reinterpret_cast<const char*>(handle), 64));
}
bool heap_open_ipc(uint64_t h, const std::string& all_handles) {
  return atomo_heap_open_ipc(P<void>(h), reinterpret_cast<const unsigned char*>(all_handles.data())) != 0;
}

torch::Tensor tensor_from_ptr(uint64_t ptr, int64_t numel, const std::string& dtype, int device) {
  auto dt = dtype == "int32"      ? torch::kInt32
            : dtype == "int64"    ? torch::kInt64
            : dtype == "uint8"    ? torch::kUInt8
            : dtype == "bfloat16" ? torch::kBFloat16
                                  : torch::kFloat32;
  auto opts = torch::TensorOptions().dtype(dt).device(torch::kCUDA, device);
  return torch::from_blob(P<void>(ptr), {numel}, [](void*) {}, opts);
}

// ---------------------------------------------------------------------------------------------- svd encode
void gram(const torch::Tensor& grad, const torch::Tensor& layers, const torch::Tensor& tiles, int ntiles,
          torch::Tensor gpart) {
  check_cuda_f32(grad, "grad");
  c10::cuda::CUDAGuard guard(grad.device());
  atomo_launch_gram(grad.data_ptr<float>(), layers.data_ptr(), tiles.data_ptr(), ntiles, gpart.data_ptr<float>(),
                    cur_stream());
}

void eig_sample(const torch::Tensor& layers, const torch::Tensor& ts_layers, const torch::Tensor& gpart,
                torch::Tensor vsel, torch::Tensor selcount, c10::optional<torch::Tensor> sigma_out,
                uint64_t ps_arena_peer, int64_t arena_floats, const torch::Tensor& ctrl,
                c10::optional<torch::Tensor> ext_uniforms, int rank, bool random_sample, bool waterfill,
                bool systematic, int worker_index, int threads) {
  c10::cuda::CUDAGuard guard(gpart.device());
  atomo_launch_eig_sample(layers.data_ptr(), ts_layers.data_ptr<int>(), (int)ts_layers.numel(),
                          gpart.data_ptr<float>(), vsel.data_ptr<float>(), selcount.data_ptr<int>(),
                          sigma_out.has_value() ? sigma_out->data_ptr<float>() : nullptr, P<float>(ps_arena_peer),
                          arena_floats, ctrl.data_ptr(),
                          ext_uniforms.has_value() ? ext_uniforms->data_ptr<float>() : nullptr, rank,
                          random_sample, waterfill, systematic, worker_index, threads, cur_stream());
}

void project_push(const torch::Tensor& grad, const torch::Tensor& layers, const torch::Tensor& tiles, int ntiles,
                  const torch::Tensor& vsel, const torch::Tensor& selcount, uint64_t ps_arena_peer,
                  int64_t arena_floats, uint64_t push_flag_peer, torch::Tensor ctrl, int worker_index, bool signal) {
  check_cuda_f32(grad, "grad");
  c10::cuda::CUDAGuard guard(grad.device());
  atomo_launch_project_push(grad.data_ptr<float>(), layers.data_ptr(), tiles.data_ptr(), ntiles,
                            vsel.data_ptr<float>(), selcount.data_ptr<int>(), P<float>(ps_arena_peer), arena_floats,
                            P<int>(push_flag_peer), ctrl.data_ptr(), worker_index, signal ? 1 : 0, cur_stream());
}

void signal_push(uint64_t push_flag_peer, const torch::Tensor& ctrl, int worker_index) {
  c10::cuda::CUDAGuard guard(ctrl.device());
  atomo_launch_signal_push(P<int>(push_flag_peer), ctrl.data_ptr(), worker_index, cur_stream());
}

void check_nhwc_bf16(const torch::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kBFloat16, name, " must be a CUDA bf16 tensor");
  TORCH_CHECK(t.dim() == 4 && t.is_contiguous(at::MemoryFormat::ChannelsLast), name, " must be channels_last");
  TORCH_CHECK(t.size(1) % 8 == 0 && t.size(1) <= 2048, name, ": C must be a multiple of 8 (<= 2048)");
}

// the ReLU mask of a fused BN layer: uint8, one byte (8 channel bits) per 8 channels of each row
void check_relu_mask(const torch::Tensor& mask, const torch::Tensor& x) {
  TORCH_CHECK(mask.is_cuda() && mask.scalar_type() == torch::kUInt8 && mask.is_contiguous(),
              "mask must be a contiguous CUDA uint8 tensor");
  TORCH_CHECK(mask.numel() == x.numel() / 8, "mask must hold numel(x) / 8 bytes");
}

// y = bn(x) [+ res]; with a mask, y is ReLU'd and the mask receives its y > 0 bits
void bn_forward(const torch::Tensor& x, c10::optional<torch::Tensor> res, torch::Tensor y,
                c10::optional<torch::Tensor> mask, torch::Tensor acc, const torch::Tensor& gamma,
                const torch::Tensor& beta, torch::Tensor save_mean, torch::Tensor save_invstd,
                c10::optional<torch::Tensor> running_mean, c10::optional<torch::Tensor> running_var, double eps,
                double momentum) {
  check_nhwc_bf16(x, "x");
  check_nhwc_bf16(y, "y");
  if (res.has_value()) check_nhwc_bf16(*res, "residual");
  if (mask.has_value()) check_relu_mask(*mask, x);
  c10::cuda::CUDAGuard guard(x.device());
  const long long R = x.numel() / x.size(1);
  // per-CTA partial sums (stream-ordered caching allocator: also valid inside a CUDA-graph capture)
  auto part = torch::empty({atomo_bn_partial_floats(R, (int)x.size(1))}, acc.options());
  atomo_launch_bn_forward(x.data_ptr(), res.has_value() ? res->data_ptr() : nullptr, y.data_ptr(),
                          mask.has_value() ? mask->data_ptr() : nullptr, R, (int)x.size(1), acc.data_ptr<float>(),
                          part.data_ptr<float>(), gamma.data_ptr<float>(), beta.data_ptr<float>(),
                          save_mean.data_ptr<float>(), save_invstd.data_ptr<float>(),
                          running_mean.has_value() ? running_mean->data_ptr<float>() : nullptr,
                          running_var.has_value() ? running_var->data_ptr<float>() : nullptr, (float)eps,
                          (float)momentum, cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// mask: the ReLU mask bn_forward wrote, or None for a layer without ReLU
void bn_backward(const torch::Tensor& dy, const torch::Tensor& x, c10::optional<torch::Tensor> mask, torch::Tensor dx,
                 c10::optional<torch::Tensor> dres, const torch::Tensor& mean, const torch::Tensor& invstd,
                 const torch::Tensor& gamma, torch::Tensor acc, torch::Tensor dgamma, torch::Tensor dbeta) {
  check_nhwc_bf16(dy, "dy");
  check_nhwc_bf16(x, "x");
  check_nhwc_bf16(dx, "dx");
  if (mask.has_value()) check_relu_mask(*mask, x);
  c10::cuda::CUDAGuard guard(x.device());
  const long long R = x.numel() / x.size(1);
  auto part = torch::empty({atomo_bn_partial_floats(R, (int)x.size(1))}, acc.options());
  atomo_launch_bn_backward(dy.data_ptr(), x.data_ptr(), mask.has_value() ? mask->data_ptr() : nullptr, dx.data_ptr(),
                           dres.has_value() ? dres->data_ptr() : nullptr, R, (int)x.size(1), mean.data_ptr<float>(),
                           invstd.data_ptr<float>(), gamma.data_ptr<float>(), acc.data_ptr<float>(),
                           part.data_ptr<float>(), dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// Backward of a convolution without bias whose weight gradient nobody on the current stream waits for: the input
// gradient (if input_grad) on the current stream, then the weight gradient (if weight_grad) on `wgrad_stream`, forked
// from the current stream after the input gradient was enqueued, so the backward chain's own GEMM is issued first.
// Both are the at::convolution_backward calls the stock autograd node makes as one, with the same algorithm choice,
// so the values are the same.  dy and x are marked as used on the wgrad stream: the caller frees them when this
// returns, and the caching allocator then keeps their blocks until the weight gradient has read them.  Whoever reads
// the weight gradient on another stream waits for the wgrad stream first.  Returns [dx, dw] (None where not asked).
std::vector<c10::optional<torch::Tensor>> conv_backward_split(const torch::Tensor& dy, const torch::Tensor& x,
                                                              const torch::Tensor& weight, std::vector<int64_t> stride,
                                                              std::vector<int64_t> padding,
                                                              std::vector<int64_t> dilation, int64_t groups,
                                                              bool input_grad, bool weight_grad,
                                                              uint64_t wgrad_stream) {
  TORCH_CHECK(dy.is_cuda() && x.is_cuda() && weight.is_cuda(), "conv_backward_split: CUDA tensors expected");
  TORCH_CHECK(wgrad_stream != 0 || !weight_grad, "conv_backward_split: a wgrad stream is required");
  c10::cuda::CUDAGuard guard(dy.device());
  const std::vector<int64_t> out_pad(stride.size(), 0);
  c10::optional<torch::Tensor> dx, dw;
  if (input_grad) {
    dx = std::get<0>(at::convolution_backward(dy, x, weight, c10::nullopt, stride, padding, dilation, false, out_pad,
                                              groups, {true, false, false}));
  }
  if (weight_grad) {
    const c10::cuda::CUDAStream cur = c10::cuda::getCurrentCUDAStream();
    const c10::cuda::CUDAStream side =
        c10::cuda::getStreamFromExternal(reinterpret_cast<cudaStream_t>(wgrad_stream), dy.device().index());
    at::cuda::CUDAEvent fork;
    fork.record(cur);
    fork.block(side);
    {
      c10::cuda::CUDAStreamGuard on_side(side);
      dw = std::get<1>(at::convolution_backward(dy, x, weight, c10::nullopt, stride, padding, dilation, false,
                                                out_pad, groups, {false, true, false}));
    }
    c10::cuda::CUDACachingAllocator::recordStream(dy.storage().data_ptr(), side);
    c10::cuda::CUDACachingAllocator::recordStream(x.storage().data_ptr(), side);
  }
  return {dx, dw};
}

void skinny_gemm(const torch::Tensor& tiles, int ntiles, torch::Tensor ctrl, int grid) {
  c10::cuda::CUDAGuard guard(tiles.device());
  atomo_launch_skinny_gemm(tiles.data_ptr(), ntiles, ctrl.data_ptr(), grid, cur_stream());
}

void ext_finalize(const torch::Tensor& descs, const torch::Tensor& tiles, int ntiles, const torch::Tensor& arena_y,
                  const torch::Tensor& arena_b, uint64_t ps_arena_peer, int64_t arena_floats,
                  const torch::Tensor& ctrl, int worker_index) {
  check_cuda_f32(arena_y, "arena_y");
  c10::cuda::CUDAGuard guard(arena_y.device());
  atomo_launch_ext_finalize(descs.data_ptr(), tiles.data_ptr(), ntiles, arena_y.data_ptr<float>(),
                            arena_b.data_ptr<float>(), P<float>(ps_arena_peer), arena_floats, ctrl.data_ptr(),
                            worker_index, cur_stream());
}

// ---------------------------------------------------------------------------------------------- PS
void ps_update(const torch::Tensor& layers, const torch::Tensor& tiles, int ntiles, int W, int nflags, int nranks,
               torch::Tensor params, torch::Tensor momentum, const torch::Tensor& params_peer, uint64_t params_mc,
               const torch::Tensor& grads_peer, uint64_t grads_mc, uint64_t arenas, int64_t arena_floats,
               uint64_t push_flags, const torch::Tensor& param_flag_peer, torch::Tensor ctrl,
               int64_t timeout_ticks, double inv_w, int grid, uint64_t tstats) {
  check_cuda_f32(params, "params");
  check_cuda_f32(momentum, "momentum");
  TORCH_CHECK(W <= atomo_ps_max_workers(), "too many workers for ps_update");
  c10::cuda::CUDAGuard guard(params.device());
  atomo_launch_ps_update(layers.data_ptr(), tiles.data_ptr(), ntiles, W, nflags, nranks, params.data_ptr<float>(),
                         momentum.data_ptr<float>(), reinterpret_cast<float* const*>(params_peer.data_ptr()),
                         P<float>(params_mc), reinterpret_cast<const float* const*>(grads_peer.data_ptr()),
                         P<const float>(grads_mc), P<const float>(arenas), arena_floats, P<int>(push_flags),
                         reinterpret_cast<int* const*>(param_flag_peer.data_ptr()), ctrl.data_ptr(), timeout_ticks,
                         (float)inv_w, grid, P<long long>(tstats), cur_stream());
}

void wait_params(uint64_t param_flag, torch::Tensor ctrl, int64_t timeout_ticks, uint64_t tstats) {
  c10::cuda::CUDAGuard guard(ctrl.device());
  atomo_launch_wait_params(P<const int>(param_flag), ctrl.data_ptr(), timeout_ticks, P<long long>(tstats),
                           cur_stream());
}
void advance_step(torch::Tensor ctrl) {
  c10::cuda::CUDAGuard guard(ctrl.device());
  atomo_launch_advance_step(ctrl.data_ptr(), cur_stream());
}
void param_bcast(const torch::Tensor& src, const torch::Tensor& params_peer, uint64_t params_mc, int nranks,
                 int self_rank, int64_t numel) {
  check_cuda_f32(src, "src");
  c10::cuda::CUDAGuard guard(src.device());
  atomo_launch_param_bcast(src.data_ptr<float>(), reinterpret_cast<float* const*>(params_peer.data_ptr()),
                           P<float>(params_mc), nranks, self_rank, numel, cur_stream());
}
void set_flags(const torch::Tensor& flag_peer, int nranks, int value) {
  c10::cuda::CUDAGuard guard(flag_peer.device());
  atomo_launch_set_flags(reinterpret_cast<int* const*>(flag_peer.data_ptr()), nranks, value, cur_stream());
}

// ---------------------------------------------------------------------------------------------- qsgd / entrywise
void qsgd_encode(const torch::Tensor& grad, int64_t numel, int bucket, int q, bool terngrad,
                 c10::optional<torch::Tensor> clip, uint64_t words_out, uint64_t norms_out,
                 const torch::Tensor& ctrl, int worker_index, c10::optional<torch::Tensor> ext_uniforms) {
  check_cuda_f32(grad, "grad");
  TORCH_CHECK(q >= 1 && q <= 14, "GPU QSGD supports quantization_level in [1, 14]");
  TORCH_CHECK(bucket >= 32 && bucket <= atomo_qsgd_max_bucket(), "bucket_size out of range for the GPU path");
  c10::cuda::CUDAGuard guard(grad.device());
  atomo_launch_qsgd_encode(grad.data_ptr<float>(), numel, bucket, q, terngrad,
                           clip.has_value() ? clip->data_ptr<float>() : nullptr, P<unsigned long long>(words_out),
                           P<float>(norms_out), ctrl.data_ptr(), worker_index,
                           ext_uniforms.has_value() ? ext_uniforms->data_ptr<float>() : nullptr, cur_stream());
}
void qsgd_decode_sum(const torch::Tensor& words_ptrs, const torch::Tensor& norms_ptrs, int W, int64_t numel,
                     int bucket, int q, bool terngrad, torch::Tensor out_sum, uint64_t push_flags,
                     torch::Tensor ctrl, int64_t timeout_ticks) {
  check_cuda_f32(out_sum, "out_sum");
  c10::cuda::CUDAGuard guard(out_sum.device());
  atomo_launch_qsgd_decode_sum(reinterpret_cast<const unsigned long long* const*>(words_ptrs.data_ptr()),
                               reinterpret_cast<const float* const*>(norms_ptrs.data_ptr()), W, numel, bucket, q,
                               terngrad, out_sum.data_ptr<float>(), P<const int>(push_flags), ctrl.data_ptr(),
                               timeout_ticks, cur_stream());
}
void entrywise_encode(const torch::Tensor& grad, const torch::Tensor& layers, const torch::Tensor& tiles,
                      int ntiles, torch::Tensor l1, double budget, uint64_t idx_out, uint64_t val_out,
                      uint64_t count_out, int capacity, torch::Tensor local_count, uint64_t push_flag_peer,
                      torch::Tensor ctrl, int worker_index, c10::optional<torch::Tensor> ext_uniforms, bool signal) {
  check_cuda_f32(grad, "grad");
  c10::cuda::CUDAGuard guard(grad.device());
  atomo_launch_entrywise_encode(grad.data_ptr<float>(), layers.data_ptr(), tiles.data_ptr(), ntiles,
                                l1.data_ptr<float>(), (int)l1.numel(), (float)budget, P<int>(idx_out),
                                P<float>(val_out), P<int>(count_out), capacity, local_count.data_ptr<int>(),
                                P<int>(push_flag_peer), ctrl.data_ptr(), worker_index,
                                ext_uniforms.has_value() ? ext_uniforms->data_ptr<float>() : nullptr,
                                signal ? 1 : 0, cur_stream());
}
void entrywise_scatter(const torch::Tensor& idx_ptrs, const torch::Tensor& val_ptrs, const torch::Tensor& count_ptrs,
                       int W, int capacity, torch::Tensor out_sum, int64_t numel, uint64_t push_flags,
                       torch::Tensor ctrl, int64_t timeout_ticks) {
  check_cuda_f32(out_sum, "out_sum");
  c10::cuda::CUDAGuard guard(out_sum.device());
  atomo_launch_entrywise_scatter(reinterpret_cast<const int* const*>(idx_ptrs.data_ptr()),
                                 reinterpret_cast<const float* const*>(val_ptrs.data_ptr()),
                                 reinterpret_cast<const int* const*>(count_ptrs.data_ptr()), W, capacity,
                                 out_sum.data_ptr<float>(), numel, P<const int>(push_flags), ctrl.data_ptr(),
                                 timeout_ticks, cur_stream());
}

// ---------------------------------------------------------------------------------------------- v2 engine
// Every pointer argument is a raw device address (uint64): the engine keeps the tensors alive.
void v2_encode(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t gpart, uint64_t counters,
               uint64_t vsel, uint64_t selcount, uint64_t sigma_out, uint64_t arena_peer, int n_owners,
               int64_t arena_floats, uint64_t stage, uint64_t ctrl, uint64_t ext_uniforms, uint64_t vprev,
               int max_sweeps, bool random_sample, bool waterfill, bool systematic, int worker,
               bool resample_empty, int flags, uint64_t tstats, int group) {
  atomo_v2_launch_encode(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                         P<float>(gpart), P<unsigned int>(counters), P<float>(vsel), P<int>(selcount),
                         P<float>(sigma_out), P<float* const>(arena_peer), n_owners, arena_floats, P<void>(stage),
                         P<const void>(ctrl), P<const float>(ext_uniforms), P<float>(vprev), max_sweeps, random_sample,
                         waterfill, systematic, worker, resample_empty ? 1 : 0, flags, P<long long>(tstats), group,
                         cur_stream());
}
void v2_project(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t vsel, uint64_t selcount,
                uint64_t arena_peer, uint64_t sig_peer, int n_owners, int64_t arena_floats, int worker, int group,
                uint64_t ctrl, uint64_t group_counter, int flags, uint64_t tstats, bool final_group, bool timed,
                uint64_t residual, int ef_owner) {
  TORCH_CHECK(residual == 0 || (ef_owner >= 0 && ef_owner < n_owners), "v2_project: ef_owner must be an owner index");
  atomo_v2_launch_project(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                          P<const float>(vsel), P<const int>(selcount), P<float* const>(arena_peer),
                          P<int* const>(sig_peer), n_owners, arena_floats, worker, group, P<void>(ctrl),
                          P<unsigned int>(group_counter), flags, P<long long>(tstats), final_group ? 1 : 0,
                          timed ? 1 : 0, P<float>(residual), ef_owner, cur_stream());
}
void v2_ps(uint64_t units, uint64_t tiles, int tile0, int ntiles, int W, int nranks, int group, bool final_group,
           int owner, uint64_t master, uint64_t mom, uint64_t sq, uint64_t sqmax, uint64_t vmom, uint64_t vsq,
           uint64_t vsqmax, uint64_t wshadow_mc, uint64_t wshadow_peer, uint64_t vparams_local, uint64_t vparams_mc,
           uint64_t vparams_peer, uint64_t vgrads_mc, uint64_t vgrads_peer, uint64_t stage_peer, uint64_t arenas,
           int64_t arena_floats, uint64_t sig, uint64_t sig_peer, uint64_t ctrl, uint64_t group_counter,
           int64_t timeout, uint64_t tstats, double inv_w, int grid) {
  TORCH_CHECK(W <= 16, "too many workers for v2_ps");
  atomo_v2_launch_ps(P<const void>(units), P<const void>(tiles), tile0, ntiles, W, nranks, group, final_group ? 1 : 0,
                     owner, P<float>(master), P<float>(mom), P<float>(sq), P<float>(sqmax), P<float>(vmom),
                     P<float>(vsq), P<float>(vsqmax), P<void>(wshadow_mc), P<void* const>(wshadow_peer),
                     P<float>(vparams_local), P<float>(vparams_mc), P<float* const>(vparams_peer),
                     P<const float>(vgrads_mc), P<const float* const>(vgrads_peer), P<const void* const>(stage_peer),
                     P<const float>(arenas), arena_floats, P<int>(sig), P<int* const>(sig_peer), P<void>(ctrl),
                     P<unsigned int>(group_counter), timeout, P<long long>(tstats), (float)inv_w, grid, cur_stream());
}
// QSGD / TernGrad: q and the bucket travel in the unit table; `max_level` / `max_bucket` are the largest values the
// plan holds (checked here against what the kernels can represent)
void check_qsgd_plan(int max_level, int max_bucket) {
  TORCH_CHECK(max_level >= 1 && max_level <= 14, "v2 QSGD: quantization_level must be in [1, 14]");
  TORCH_CHECK(max_bucket >= 1 && max_bucket <= 1024, "v2 QSGD: bucket must be in [1, 1024]");
}
void v2_qsgd_stats(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t partials,
                   uint64_t counters, uint64_t clip, uint64_t tstats, int group) {
  TORCH_CHECK(partials != 0 && clip != 0 && counters != 0, "v2_qsgd_stats: partials / counters / clip required");
  atomo_v2_launch_qsgd_stats(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                             P<double>(partials), P<unsigned int>(counters), P<float>(clip), P<long long>(tstats),
                             group, cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_qsgd_encode(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t clip,
                    uint64_t arena_peer, uint64_t sig_peer, int n_owners, int64_t arena_floats, int worker, int group,
                    uint64_t ctrl, uint64_t group_counter, uint64_t ext_uniforms, uint64_t tstats, bool final_group,
                    bool stamp_start, int max_level, int max_bucket, bool terngrad, uint64_t residual) {
  check_qsgd_plan(max_level, max_bucket);
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_qsgd_encode: worker index must be in [0, 16)");
  TORCH_CHECK(!terngrad || clip != 0, "v2_qsgd_encode: TernGrad needs the clip buffer of v2_qsgd_stats");
  TORCH_CHECK(!terngrad || residual == 0, "v2_qsgd_encode: no error feedback for TernGrad (the owners rescale every "
              "worker by the shared max norm)");
  atomo_v2_launch_qsgd_encode(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                              P<const float>(clip), P<float* const>(arena_peer), P<int* const>(sig_peer), n_owners,
                              arena_floats, worker, group, P<const void>(ctrl), P<unsigned int>(group_counter),
                              P<const float>(ext_uniforms), P<long long>(tstats), final_group ? 1 : 0,
                              stamp_start ? 1 : 0, P<float>(residual), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_ps_qsgd(uint64_t units, uint64_t tiles, int tile0, int ntiles, int W, int nranks, int group, bool final_group,
                int owner, uint64_t master, uint64_t mom, uint64_t sq, uint64_t sqmax, uint64_t vmom, uint64_t vsq,
                uint64_t vsqmax, uint64_t wshadow_mc, uint64_t wshadow_peer, uint64_t vparams_local,
                uint64_t vparams_mc, uint64_t vparams_peer, uint64_t vgrads_mc, uint64_t vgrads_peer, uint64_t arenas,
                int64_t arena_floats, uint64_t sig, uint64_t sig_peer, uint64_t ctrl, uint64_t group_counter,
                int64_t timeout, uint64_t tstats, double inv_w, int grid, int max_level, int max_bucket) {
  TORCH_CHECK(W >= 1 && W <= 16, "too many workers for v2_ps_qsgd");
  check_qsgd_plan(max_level, max_bucket);
  atomo_v2_launch_ps_qsgd(P<const void>(units), P<const void>(tiles), tile0, ntiles, W, nranks, group,
                          final_group ? 1 : 0, owner, P<float>(master), P<float>(mom), P<float>(sq), P<float>(sqmax),
                          P<float>(vmom), P<float>(vsq), P<float>(vsqmax), P<void>(wshadow_mc),
                          P<void* const>(wshadow_peer), P<float>(vparams_local), P<float>(vparams_mc),
                          P<float* const>(vparams_peer), P<const float>(vgrads_mc), P<const float* const>(vgrads_peer),
                          P<const float>(arenas), arena_floats, P<int>(sig), P<int* const>(sig_peer), P<void>(ctrl),
                          P<unsigned int>(group_counter), timeout, P<long long>(tstats), (float)inv_w, grid,
                          cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
// entry-wise ATOMO: the budget travels in the unit table, the L1 norms (fp64, one per entry unit) between the launches
void v2_entry_stats(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t partials,
                    uint64_t counters, uint64_t l1, uint64_t tstats, int group) {
  TORCH_CHECK(partials != 0 && l1 != 0 && counters != 0, "v2_entry_stats: partials / counters / l1 required");
  atomo_v2_launch_entry_stats(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                              P<double>(partials), P<unsigned int>(counters), P<double>(l1), P<long long>(tstats),
                              group, cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_entry_encode(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t l1,
                     uint64_t arena_peer, uint64_t sig_peer, int n_owners, int64_t arena_floats, int worker, int group,
                     uint64_t ctrl, uint64_t group_counter, uint64_t ext_uniforms, uint64_t tstats, bool final_group,
                     uint64_t residual) {
  TORCH_CHECK(l1 != 0, "v2_entry_encode: needs the L1 norms of v2_entry_stats");
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_entry_encode: worker index must be in [0, 16)");
  atomo_v2_launch_entry_encode(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                               P<const double>(l1), P<float* const>(arena_peer), P<int* const>(sig_peer), n_owners,
                               arena_floats, worker, group, P<const void>(ctrl), P<unsigned int>(group_counter),
                               P<const float>(ext_uniforms), P<long long>(tstats), final_group ? 1 : 0,
                               P<float>(residual), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
// top-k: the two selection launches (high / low magnitude bits; per-unit histogram, tile counts, state) of one group
void v2_topk_select(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t hist,
                    uint64_t tile_counts, uint64_t counters, uint64_t sel, uint64_t tstats, int group) {
  TORCH_CHECK(hist != 0 && tile_counts != 0 && counters != 0 && sel != 0,
              "v2_topk_select: hist / tile_counts / counters / sel required");
  atomo_v2_launch_topk_select(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                              P<int>(hist), P<int>(tile_counts), P<unsigned int>(counters), P<int>(sel),
                              P<long long>(tstats), group, cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_topk_encode(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t sel,
                    uint64_t tile_counts, uint64_t arena_peer, uint64_t sig_peer, int n_owners, int64_t arena_floats,
                    int worker, int group, uint64_t ctrl, uint64_t group_counter, uint64_t tstats, bool final_group,
                    uint64_t residual) {
  TORCH_CHECK(sel != 0 && tile_counts != 0, "v2_topk_encode: needs the selection of v2_topk_select");
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_topk_encode: worker index must be in [0, 16)");
  atomo_v2_launch_topk_encode(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                              P<const int>(sel), P<const int>(tile_counts), P<float* const>(arena_peer),
                              P<int* const>(sig_peer), n_owners, arena_floats, worker, group, P<const void>(ctrl),
                              P<unsigned int>(group_counter), P<long long>(tstats), final_group ? 1 : 0,
                              P<float>(residual), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_topk_code_stats(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t sel,
                        uint64_t tile_counts, uint64_t arena_peer, int n_owners, int64_t arena_floats, int worker,
                        uint64_t partials, uint64_t counters, uint64_t acc) {
  TORCH_CHECK(partials != 0 && counters != 0 && acc != 0 && sel != 0 && tile_counts != 0,
              "v2_topk_code_stats: partials / counters / acc / sel / tile_counts required");
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_topk_code_stats: worker index must be in [0, 16)");
  atomo_v2_launch_topk_code_stats(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                                  P<const int>(sel), P<const int>(tile_counts), P<float* const>(arena_peer), n_owners,
                                  arena_floats, worker, P<double>(partials), P<unsigned int>(counters), P<double>(acc),
                                  cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
// scaled sign: the bucket travels in the unit table; the encode is the group's only launch (it raises the push flag)
void v2_sign_encode(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t arena_peer,
                    uint64_t sig_peer, int n_owners, int64_t arena_floats, int worker, int group, uint64_t ctrl,
                    uint64_t group_counter, uint64_t tstats, bool final_group, uint64_t residual) {
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_sign_encode: worker index must be in [0, 16)");
  atomo_v2_launch_sign_encode(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                              P<float* const>(arena_peer), P<int* const>(sig_peer), n_owners, arena_floats, worker,
                              group, P<const void>(ctrl), P<unsigned int>(group_counter), P<long long>(tstats),
                              final_group ? 1 : 0, P<float>(residual), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_ps_sign(uint64_t units, uint64_t tiles, int tile0, int ntiles, int W, int nranks, int group, bool final_group,
                int owner, uint64_t master, uint64_t mom, uint64_t sq, uint64_t sqmax, uint64_t vmom, uint64_t vsq,
                uint64_t vsqmax, uint64_t wshadow_mc, uint64_t wshadow_peer, uint64_t vparams_local,
                uint64_t vparams_mc, uint64_t vparams_peer, uint64_t vgrads_mc, uint64_t vgrads_peer, uint64_t arenas,
                int64_t arena_floats, uint64_t sig, uint64_t sig_peer, uint64_t ctrl, uint64_t group_counter,
                int64_t timeout, uint64_t tstats, double inv_w, int grid) {
  TORCH_CHECK(W >= 1 && W <= 16, "too many workers for v2_ps_sign");
  atomo_v2_launch_ps_sign(P<const void>(units), P<const void>(tiles), tile0, ntiles, W, nranks, group,
                          final_group ? 1 : 0, owner, P<float>(master), P<float>(mom), P<float>(sq), P<float>(sqmax),
                          P<float>(vmom), P<float>(vsq), P<float>(vsqmax), P<void>(wshadow_mc),
                          P<void* const>(wshadow_peer), P<float>(vparams_local), P<float>(vparams_mc),
                          P<float* const>(vparams_peer), P<const float>(vgrads_mc), P<const float* const>(vgrads_peer),
                          P<const float>(arenas), arena_floats, P<int>(sig), P<int* const>(sig_peer), P<void>(ctrl),
                          P<unsigned int>(group_counter), timeout, P<long long>(tstats), (float)inv_w, grid,
                          cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_sign_code_stats(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t arena_peer,
                        int n_owners, int64_t arena_floats, int worker, uint64_t partials, uint64_t counters,
                        uint64_t acc) {
  TORCH_CHECK(partials != 0 && counters != 0 && acc != 0, "v2_sign_code_stats: partials / counters / acc required");
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_sign_code_stats: worker index must be in [0, 16)");
  atomo_v2_launch_sign_code_stats(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                                  P<float* const>(arena_peer), n_owners, arena_floats, worker, P<double>(partials),
                                  P<unsigned int>(counters), P<double>(acc), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
// fp8: the bucket travels in the unit table; the encode is the group's only launch (it raises the push flag)
void v2_fp8_encode(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t arena_peer,
                   uint64_t sig_peer, int n_owners, int64_t arena_floats, int worker, int group, uint64_t ctrl,
                   uint64_t group_counter, uint64_t tstats, bool final_group, uint64_t residual) {
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_fp8_encode: worker index must be in [0, 16)");
  atomo_v2_launch_fp8_encode(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                             P<float* const>(arena_peer), P<int* const>(sig_peer), n_owners, arena_floats, worker,
                             group, P<const void>(ctrl), P<unsigned int>(group_counter), P<long long>(tstats),
                             final_group ? 1 : 0, P<float>(residual), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_ps_fp8(uint64_t units, uint64_t tiles, int tile0, int ntiles, int W, int nranks, int group, bool final_group,
               int owner, uint64_t master, uint64_t mom, uint64_t sq, uint64_t sqmax, uint64_t vmom, uint64_t vsq,
               uint64_t vsqmax, uint64_t wshadow_mc, uint64_t wshadow_peer, uint64_t vparams_local,
               uint64_t vparams_mc, uint64_t vparams_peer, uint64_t vgrads_mc, uint64_t vgrads_peer, uint64_t arenas,
               int64_t arena_floats, uint64_t sig, uint64_t sig_peer, uint64_t ctrl, uint64_t group_counter,
               int64_t timeout, uint64_t tstats, double inv_w, int grid) {
  TORCH_CHECK(W >= 1 && W <= 16, "too many workers for v2_ps_fp8");
  atomo_v2_launch_ps_fp8(P<const void>(units), P<const void>(tiles), tile0, ntiles, W, nranks, group,
                         final_group ? 1 : 0, owner, P<float>(master), P<float>(mom), P<float>(sq), P<float>(sqmax),
                         P<float>(vmom), P<float>(vsq), P<float>(vsqmax), P<void>(wshadow_mc),
                         P<void* const>(wshadow_peer), P<float>(vparams_local), P<float>(vparams_mc),
                         P<float* const>(vparams_peer), P<const float>(vgrads_mc), P<const float* const>(vgrads_peer),
                         P<const float>(arenas), arena_floats, P<int>(sig), P<int* const>(sig_peer), P<void>(ctrl),
                         P<unsigned int>(group_counter), timeout, P<long long>(tstats), (float)inv_w, grid,
                         cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_fp8_code_stats(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t arena_peer,
                       int n_owners, int64_t arena_floats, int worker, uint64_t partials, uint64_t counters,
                       uint64_t acc) {
  TORCH_CHECK(partials != 0 && counters != 0 && acc != 0, "v2_fp8_code_stats: partials / counters / acc required");
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_fp8_code_stats: worker index must be in [0, 16)");
  atomo_v2_launch_fp8_code_stats(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                                 P<float* const>(arena_peer), n_owners, arena_floats, worker, P<double>(partials),
                                 P<unsigned int>(counters), P<double>(acc), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
// PowerSGD: Q_w of every unit drawn once (draw 0), outside the captured graph
void v2_powersgd_init(uint64_t units, int n_units, uint64_t scratch, uint64_t ctrl) {
  TORCH_CHECK(scratch != 0 && ctrl != 0, "v2_powersgd_init: scratch / ctrl required");
  atomo_v2_launch_powersgd_init(P<const void>(units), n_units, P<float>(scratch), P<const void>(ctrl), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
// PowerSGD encode of one backward group: pass A over the encode tiles, pass B over the pw tiles (it raises the push
// flag), then the error-feedback pass when a residual is given
void v2_powersgd_encode(uint64_t units, uint64_t enc_tiles, int tile0, int ntiles, uint64_t pw_tiles, int pw0, int npw,
                        uint64_t gptr, uint64_t scratch, uint64_t gram, uint64_t state, uint64_t stage,
                        uint64_t arena_peer, uint64_t sig_peer, int n_owners, int64_t arena_floats, int worker,
                        int group, uint64_t ctrl, uint64_t group_counter, uint64_t tstats, bool final_group,
                        uint64_t residual) {
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_powersgd_encode: worker index must be in [0, 16)");
  TORCH_CHECK(scratch != 0 && gram != 0 && state != 0, "v2_powersgd_encode: scratch / gram / state required");
  atomo_v2_launch_powersgd_encode(P<const void>(units), P<const void>(enc_tiles), tile0, ntiles, P<const void>(pw_tiles),
                                  pw0, npw, P<const long long>(gptr), P<float>(scratch), P<double>(gram), P<void>(state),
                                  P<void>(stage), P<float* const>(arena_peer), P<int* const>(sig_peer), n_owners,
                                  arena_floats, worker, group, P<const void>(ctrl), P<unsigned int>(group_counter),
                                  P<long long>(tstats), final_group ? 1 : 0, P<float>(residual), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_ps_powersgd(uint64_t units, uint64_t tiles, int tile0, int ntiles, int W, int nranks, int group,
                    bool final_group, int owner, uint64_t master, uint64_t mom, uint64_t sq, uint64_t sqmax,
                    uint64_t vmom, uint64_t vsq, uint64_t vsqmax, uint64_t wshadow_mc, uint64_t wshadow_peer,
                    uint64_t vparams_local, uint64_t vparams_mc, uint64_t vparams_peer, uint64_t vgrads_mc,
                    uint64_t vgrads_peer, uint64_t stage_peer, uint64_t arenas, int64_t arena_floats, uint64_t sig,
                    uint64_t sig_peer, uint64_t ctrl, uint64_t group_counter, int64_t timeout, uint64_t tstats,
                    double inv_w, int grid) {
  TORCH_CHECK(W >= 1 && W <= 16, "too many workers for v2_ps_powersgd");
  atomo_v2_launch_ps_powersgd(P<const void>(units), P<const void>(tiles), tile0, ntiles, W, nranks, group,
                              final_group ? 1 : 0, owner, P<float>(master), P<float>(mom), P<float>(sq),
                              P<float>(sqmax), P<float>(vmom), P<float>(vsq), P<float>(vsqmax), P<void>(wshadow_mc),
                              P<void* const>(wshadow_peer), P<float>(vparams_local), P<float>(vparams_mc),
                              P<float* const>(vparams_peer), P<const float>(vgrads_mc),
                              P<const float* const>(vgrads_peer), P<const void* const>(stage_peer),
                              P<const float>(arenas), arena_floats, P<int>(sig), P<int* const>(sig_peer),
                              P<void>(ctrl), P<unsigned int>(group_counter), timeout, P<long long>(tstats),
                              (float)inv_w, grid, cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_powersgd_code_stats(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t scratch,
                            uint64_t state, uint64_t partials, uint64_t counters, uint64_t acc) {
  TORCH_CHECK(partials != 0 && counters != 0 && acc != 0, "v2_powersgd_code_stats: partials / counters / acc required");
  atomo_v2_launch_powersgd_code_stats(P<const void>(units), P<const void>(tiles), tile0, ntiles,
                                      P<const long long>(gptr), P<float>(scratch), P<const void>(state),
                                      P<double>(partials), P<unsigned int>(counters), P<double>(acc), cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
// error feedback: A = g + e, bf16(A) into the gradient buffers, A - bf16(A) into the residual, for the apply chunks
// [chunk0, chunk0 + nchunks) of the chunk table (one backward group); before the group's encode, on the same stream
void v2_ef_apply(uint64_t chunks, int chunk0, int nchunks, uint64_t gptr, uint64_t residual) {
  TORCH_CHECK(chunks != 0 && gptr != 0 && residual != 0, "v2_ef_apply: chunks / gptr / residual required");
  atomo_v2_launch_ef_apply(P<const void>(chunks), chunk0, nchunks, P<const long long>(gptr), P<float>(residual),
                           cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
// estimator statistics of one group: after the group's push, on the same stream
void v2_code_stats(uint64_t units, uint64_t tiles, int tile0, int ntiles, uint64_t gptr, uint64_t sigma,
                   uint64_t selcount, uint64_t l1, uint64_t clip, uint64_t arena_peer, int n_owners,
                   int64_t arena_floats, int worker, bool random_sample, bool waterfill, uint64_t partials,
                   uint64_t counters, uint64_t acc) {
  TORCH_CHECK(partials != 0 && counters != 0 && acc != 0, "v2_code_stats: partials / counters / acc required");
  TORCH_CHECK(worker >= 0 && worker < 16, "v2_code_stats: worker index must be in [0, 16)");
  atomo_v2_launch_code_stats(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                             P<const float>(sigma), P<const int>(selcount), P<const double>(l1), P<const float>(clip),
                             P<float* const>(arena_peer), n_owners, arena_floats, worker, random_sample ? 1 : 0,
                             waterfill ? 1 : 0, P<double>(partials), P<unsigned int>(counters), P<double>(acc),
                             cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_ps_entry(uint64_t units, uint64_t tiles, int tile0, int ntiles, int W, int nranks, int group, bool final_group,
                 int owner, uint64_t master, uint64_t mom, uint64_t sq, uint64_t sqmax, uint64_t vmom, uint64_t vsq,
                 uint64_t vsqmax, uint64_t wshadow_mc, uint64_t wshadow_peer, uint64_t vparams_local,
                 uint64_t vparams_mc, uint64_t vparams_peer, uint64_t vgrads_mc, uint64_t vgrads_peer, uint64_t arenas,
                 int64_t arena_floats, uint64_t sig, uint64_t sig_peer, uint64_t ctrl, uint64_t group_counter,
                 int64_t timeout, uint64_t tstats, double inv_w, int grid) {
  TORCH_CHECK(W >= 1 && W <= 16, "too many workers for v2_ps_entry");
  atomo_v2_launch_ps_entry(P<const void>(units), P<const void>(tiles), tile0, ntiles, W, nranks, group,
                           final_group ? 1 : 0, owner, P<float>(master), P<float>(mom), P<float>(sq), P<float>(sqmax),
                           P<float>(vmom), P<float>(vsq), P<float>(vsqmax), P<void>(wshadow_mc),
                           P<void* const>(wshadow_peer), P<float>(vparams_local), P<float>(vparams_mc),
                           P<float* const>(vparams_peer), P<const float>(vgrads_mc), P<const float* const>(vgrads_peer),
                           P<const float>(arenas), arena_floats, P<int>(sig), P<int* const>(sig_peer), P<void>(ctrl),
                           P<unsigned int>(group_counter), timeout, P<long long>(tstats), (float)inv_w, grid,
                           cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}
void v2_wait_params(uint64_t sig, int n_owners, uint64_t ctrl, int64_t timeout, uint64_t tstats) {
  atomo_v2_launch_wait_params(P<const int>(sig), n_owners, P<void>(ctrl), timeout, P<long long>(tstats), cur_stream());
}
void v2_advance_step(uint64_t ctrl) { atomo_v2_launch_advance_step(P<void>(ctrl), cur_stream()); }
void v2_bcast_bytes(uint64_t src, uint64_t peer, uint64_t mc, int nranks, int self, int64_t nbytes) {
  atomo_v2_launch_bcast_bytes(P<const void>(src), P<void* const>(peer), P<void>(mc), nranks, self, nbytes,
                              cur_stream());
}

// ---------------------------------------------------------------------------------------------- training input
// src [N, H, W, C] uint8 or fp32, labels [N] int64, order int32 (the epoch's sample order), mean_std [2, C] fp32,
// ext_draws [B, 3] int32 (tests); writes x [B, C, H, W] fp32 at its own strides and y [B] int64.
void augment_gather(const torch::Tensor& src, const torch::Tensor& labels, const torch::Tensor& order, int64_t pos0,
                    const torch::Tensor& mean_std, int pad, bool reflect, bool augment, uint64_t seed, int64_t epoch,
                    c10::optional<torch::Tensor> ext_draws, torch::Tensor x, torch::Tensor y) {
  TORCH_CHECK(src.is_cuda() && src.dim() == 4 && src.is_contiguous(), "src must be a contiguous CUDA [N, H, W, C]");
  const bool u8 = src.scalar_type() == torch::kUInt8;
  TORCH_CHECK(u8 || src.scalar_type() == torch::kFloat32, "src must be uint8 or float32");
  const int64_t N = src.size(0), H = src.size(1), W = src.size(2), C = src.size(3);
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == torch::kFloat32 && x.dim() == 4, "x must be a CUDA fp32 [B, C, H, W]");
  const int64_t B = x.size(0);
  TORCH_CHECK(x.size(1) == C && x.size(2) == H && x.size(3) == W, "x must be [B, C, H, W] of src's image shape");
  TORCH_CHECK(y.is_cuda() && y.scalar_type() == torch::kInt64 && y.is_contiguous() && y.numel() == B,
              "y must be a contiguous CUDA int64 [B]");
  TORCH_CHECK(labels.is_cuda() && labels.scalar_type() == torch::kInt64 && labels.is_contiguous() &&
                  labels.numel() == N, "labels must be a contiguous CUDA int64 [N]");
  TORCH_CHECK(order.is_cuda() && order.scalar_type() == torch::kInt32 && order.is_contiguous(),
              "order must be a contiguous CUDA int32 tensor");
  TORCH_CHECK(pos0 >= 0 && pos0 + B <= order.numel(), "the batch runs past the end of the order");
  TORCH_CHECK(mean_std.is_cuda() && mean_std.scalar_type() == torch::kFloat32 && mean_std.is_contiguous() &&
                  mean_std.numel() == 2 * C, "mean_std must be a contiguous CUDA fp32 [2, C]");
  TORCH_CHECK(pad >= 0 && (!u8 || !reflect || (pad < H && pad < W)), "reflect padding needs pad < H and pad < W");
  TORCH_CHECK(u8 || (pad == 0 && !augment), "fp32 sources are gathered without augmentation");
  if (ext_draws.has_value()) {
    TORCH_CHECK(ext_draws->is_cuda() && ext_draws->scalar_type() == torch::kInt32 && ext_draws->is_contiguous() &&
                    ext_draws->numel() == 3 * B, "ext_draws must be a contiguous CUDA int32 [B, 3]");
  }
  for (const torch::Tensor* t : std::initializer_list<const torch::Tensor*>{&labels, &order, &mean_std, &x, &y})
    TORCH_CHECK(t->device() == src.device(), "all tensors must be on src's device");
  c10::cuda::CUDAGuard guard(src.device());
  atomo_launch_augment_gather(src.data_ptr(), u8 ? 1 : 0, static_cast<const long long*>(labels.data_ptr()), (int)C,
                              (int)H, (int)W, order.data_ptr<int>(), pos0, (int)B, mean_std.data_ptr<float>(), pad,
                              reflect ? 1 : 0, augment ? 1 : 0, seed, (int)epoch,
                              ext_draws.has_value() ? ext_draws->data_ptr<int>() : nullptr, x.data_ptr<float>(),
                              x.stride(0), x.stride(1), x.stride(2), x.stride(3), static_cast<long long*>(y.data_ptr()),
                              cur_stream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "atomo_b200 native runtime: symmetric NVLink heap + sm_90a gradient-coding kernels";
  // heap
  m.def("heap_last_error", []() { return std::string(atomo_heap_last_error()); });
  m.def("heap_multicast_supported", &atomo_heap_multicast_supported);
  m.def("heap_posix_fd_supported", &atomo_heap_posix_fd_supported);
  m.def("heap_create_vmm", &heap_create_vmm);
  m.def("heap_mc_phase_a", [](uint64_t h, double t) { return atomo_heap_mc_phase_a(P<void>(h), t) != 0; });
  m.def("heap_mc_phase_b", [](uint64_t h) { return atomo_heap_mc_phase_b(P<void>(h)) != 0; });
  m.def("heap_create_ipc", &heap_create_ipc);
  m.def("heap_open_ipc", &heap_open_ipc);
  m.def("heap_ptr", [](uint64_t h, int r) { return atomo_heap_ptr(P<void>(h), r); });
  m.def("heap_mc_ptr", [](uint64_t h) { return atomo_heap_mc_ptr(P<void>(h)); });
  m.def("heap_bytes", [](uint64_t h) { return atomo_heap_bytes(P<void>(h)); });
  m.def("heap_mode", [](uint64_t h) { return std::string(atomo_heap_mode(P<void>(h))); });
  m.def("heap_destroy", [](uint64_t h) { atomo_heap_destroy(P<void>(h)); });
  m.def("tensor_from_ptr", &tensor_from_ptr);
  // kernels
  m.def("gram", &gram);
  m.def("eig_sample", &eig_sample, py::arg("layers"), py::arg("ts_layers"), py::arg("gpart"), py::arg("vsel"),
        py::arg("selcount"), py::arg("sigma_out"), py::arg("ps_arena_peer"), py::arg("arena_floats"), py::arg("ctrl"),
        py::arg("ext_uniforms"), py::arg("rank"), py::arg("random_sample"), py::arg("waterfill"),
        py::arg("systematic"), py::arg("worker_index"), py::arg("threads") = 256);
  m.def("project_push", &project_push);
  m.def("signal_push", &signal_push);
  m.def("ext_finalize", &ext_finalize);
  m.def("skinny_gemm", &skinny_gemm);
  m.def("bn_forward", &bn_forward);
  m.def("bn_backward", &bn_backward);
  m.def("conv_backward_split", &conv_backward_split);
  m.def("gemm_tile_bytes", &atomo_gemm_tile_bytes);
  m.def("gemm_smem_bytes", &atomo_gemm_smem_bytes);
  m.def("ext_desc_bytes", &atomo_ext_desc_bytes);
  m.def("ps_update", &ps_update, py::arg("layers"), py::arg("tiles"), py::arg("ntiles"), py::arg("W"),
        py::arg("nflags"), py::arg("nranks"), py::arg("params"), py::arg("momentum"), py::arg("params_peer"),
        py::arg("params_mc"), py::arg("grads_peer"), py::arg("grads_mc"), py::arg("arenas"),
        py::arg("arena_floats"), py::arg("push_flags"), py::arg("param_flag_peer"), py::arg("ctrl"),
        py::arg("timeout_ticks"), py::arg("inv_w"), py::arg("grid"), py::arg("tstats") = 0);
  m.def("wait_params", &wait_params, py::arg("param_flag"), py::arg("ctrl"), py::arg("timeout_ticks"),
        py::arg("tstats") = 0);
  m.def("advance_step", &advance_step);
  m.def("param_bcast", &param_bcast);
  m.def("set_flags", &set_flags);
  m.def("qsgd_encode", &qsgd_encode);
  m.def("qsgd_decode_sum", &qsgd_decode_sum);
  m.def("entrywise_encode", &entrywise_encode);
  m.def("entrywise_scatter", &entrywise_scatter);
  // v2 engine
  m.def("v2_encode", &v2_encode);
  // the error-feedback residual is the last argument of the encoders (0 / absent: no epilogue)
  m.def("v2_project", &v2_project, py::arg("units"), py::arg("tiles"), py::arg("tile0"), py::arg("ntiles"),
        py::arg("gptr"), py::arg("vsel"), py::arg("selcount"), py::arg("arena_peer"), py::arg("sig_peer"),
        py::arg("n_owners"), py::arg("arena_floats"), py::arg("worker"), py::arg("group"), py::arg("ctrl"),
        py::arg("group_counter"), py::arg("flags"), py::arg("tstats"), py::arg("final_group"), py::arg("timed"),
        py::arg("residual") = 0, py::arg("ef_owner") = 0);
  m.def("v2_ps", &v2_ps);
  m.def("v2_qsgd_stats", &v2_qsgd_stats);
  m.def("v2_qsgd_encode", &v2_qsgd_encode, py::arg("units"), py::arg("tiles"), py::arg("tile0"), py::arg("ntiles"),
        py::arg("gptr"), py::arg("clip"), py::arg("arena_peer"), py::arg("sig_peer"), py::arg("n_owners"),
        py::arg("arena_floats"), py::arg("worker"), py::arg("group"), py::arg("ctrl"), py::arg("group_counter"),
        py::arg("ext_uniforms"), py::arg("tstats"), py::arg("final_group"), py::arg("stamp_start"),
        py::arg("max_level"), py::arg("max_bucket"), py::arg("terngrad"), py::arg("residual") = 0);
  m.def("v2_ps_qsgd", &v2_ps_qsgd);
  m.def("v2_entry_stats", &v2_entry_stats);
  m.def("v2_entry_encode", &v2_entry_encode, py::arg("units"), py::arg("tiles"), py::arg("tile0"), py::arg("ntiles"),
        py::arg("gptr"), py::arg("l1"), py::arg("arena_peer"), py::arg("sig_peer"), py::arg("n_owners"),
        py::arg("arena_floats"), py::arg("worker"), py::arg("group"), py::arg("ctrl"), py::arg("group_counter"),
        py::arg("ext_uniforms"), py::arg("tstats"), py::arg("final_group"), py::arg("residual") = 0);
  m.def("v2_topk_select", &v2_topk_select);
  m.def("v2_topk_encode", &v2_topk_encode, py::arg("units"), py::arg("tiles"), py::arg("tile0"), py::arg("ntiles"),
        py::arg("gptr"), py::arg("sel"), py::arg("tile_counts"), py::arg("arena_peer"), py::arg("sig_peer"),
        py::arg("n_owners"), py::arg("arena_floats"), py::arg("worker"), py::arg("group"), py::arg("ctrl"),
        py::arg("group_counter"), py::arg("tstats"), py::arg("final_group"), py::arg("residual") = 0);
  m.def("v2_topk_code_stats", &v2_topk_code_stats);
  m.def("v2_topk_sizes", []() {
    return py::make_tuple(atomo_v2_topk_state_ints(), atomo_v2_topk_hist_bins(), atomo_v2_topk_tile_bins());
  });
  m.def("v2_sign_encode", &v2_sign_encode, py::arg("units"), py::arg("tiles"), py::arg("tile0"), py::arg("ntiles"),
        py::arg("gptr"), py::arg("arena_peer"), py::arg("sig_peer"), py::arg("n_owners"), py::arg("arena_floats"),
        py::arg("worker"), py::arg("group"), py::arg("ctrl"), py::arg("group_counter"), py::arg("tstats"),
        py::arg("final_group"), py::arg("residual") = 0);
  m.def("v2_ps_sign", &v2_ps_sign);
  m.def("v2_sign_code_stats", &v2_sign_code_stats);
  m.def("v2_fp8_encode", &v2_fp8_encode, py::arg("units"), py::arg("tiles"), py::arg("tile0"), py::arg("ntiles"),
        py::arg("gptr"), py::arg("arena_peer"), py::arg("sig_peer"), py::arg("n_owners"), py::arg("arena_floats"),
        py::arg("worker"), py::arg("group"), py::arg("ctrl"), py::arg("group_counter"), py::arg("tstats"),
        py::arg("final_group"), py::arg("residual") = 0);
  m.def("v2_ps_fp8", &v2_ps_fp8);
  m.def("v2_fp8_code_stats", &v2_fp8_code_stats);
  m.def("v2_powersgd_state_bytes", &atomo_v2_powersgd_state_bytes);
  m.def("v2_powersgd_init", &v2_powersgd_init);
  m.def("v2_powersgd_encode", &v2_powersgd_encode);
  m.def("v2_ps_powersgd", &v2_ps_powersgd);
  m.def("v2_powersgd_code_stats", &v2_powersgd_code_stats);
  m.def("v2_ef_apply", &v2_ef_apply);
  m.def("v2_ef_chunk_bytes", &atomo_v2_ef_chunk_bytes);
  m.def("v2_ps_entry", &v2_ps_entry);
  m.def("v2_code_stats", &v2_code_stats);
  m.def("v2_stats_fields", &atomo_v2_stats_fields);
  m.def("v2_stats_partials", &atomo_v2_stats_partials);
  m.def("v2_wait_params", &v2_wait_params);
  m.def("v2_advance_step", &v2_advance_step);
  m.def("v2_bcast_bytes", &v2_bcast_bytes);
  m.def("augment_gather", &augment_gather, py::arg("src"), py::arg("labels"), py::arg("order"), py::arg("pos0"),
        py::arg("mean_std"), py::arg("pad"), py::arg("reflect"), py::arg("augment"), py::arg("seed"),
        py::arg("epoch"), py::arg("ext_draws"), py::arg("x"), py::arg("y"));
  m.def("v2_unit_bytes", &atomo_v2_unit_bytes);
  m.def("v2_ctrl_bytes", &atomo_v2_ctrl_bytes);
  m.def("v2_enc_smem", &atomo_v2_enc_smem);
  m.def("v2_ps_smem", &atomo_v2_ps_smem);
  m.def("v2_ps_tile_elems", &atomo_v2_ps_tile_elems);
  // constants
  m.def("ps_smem_bytes", &atomo_ps_smem_bytes);
  m.def("ps_tile_elems", &atomo_ps_tile_elems);
  m.def("ps_max_rows", &atomo_ps_max_rows);
  m.def("ps_dense_elems", &atomo_ps_dense_elems);
  m.def("ps_max_workers", &atomo_ps_max_workers);
  m.def("qsgd_max_bucket", &atomo_qsgd_max_bucket);
}
