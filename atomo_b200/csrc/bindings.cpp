// Python bindings for the atomo_b200 native runtime (torch extension `atomo_b200._C`).
// Kernels live in the .cu files behind a plain C ABI; this file only adapts
// torch tensors / raw peer pointers to those launchers on the current stream.
#include <ATen/cuda/CUDAContext.h>
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
void atomo_launch_bn_forward(const void* x, const void* res, void* y, long long R, int C, float* acc, float* part,
                             const float* gamma, const float* beta, float* save_mean, float* save_invstd,
                             float* running_mean, float* running_var, float eps, float momentum, int relu,
                             cudaStream_t stream);
void atomo_launch_bn_backward(const void* dy, const void* x, const void* y, void* dx, void* dres, long long R, int C,
                              const float* mean, const float* invstd, const float* gamma, float* acc, float* part,
                              float* dgamma, float* dbeta, int relu, cudaStream_t stream);
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
                             cudaStream_t stream);
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

void bn_forward(const torch::Tensor& x, c10::optional<torch::Tensor> res, torch::Tensor y, torch::Tensor acc,
                const torch::Tensor& gamma, const torch::Tensor& beta, torch::Tensor save_mean,
                torch::Tensor save_invstd, c10::optional<torch::Tensor> running_mean,
                c10::optional<torch::Tensor> running_var, double eps, double momentum, bool relu) {
  check_nhwc_bf16(x, "x");
  check_nhwc_bf16(y, "y");
  if (res.has_value()) check_nhwc_bf16(*res, "residual");
  c10::cuda::CUDAGuard guard(x.device());
  const long long R = x.numel() / x.size(1);
  // per-CTA partial sums (stream-ordered caching allocator: also valid inside a CUDA-graph capture)
  auto part = torch::empty({atomo_bn_partial_floats(R, (int)x.size(1))}, acc.options());
  atomo_launch_bn_forward(x.data_ptr(), res.has_value() ? res->data_ptr() : nullptr, y.data_ptr(), R, (int)x.size(1),
                          acc.data_ptr<float>(), part.data_ptr<float>(), gamma.data_ptr<float>(), beta.data_ptr<float>(),
                          save_mean.data_ptr<float>(), save_invstd.data_ptr<float>(),
                          running_mean.has_value() ? running_mean->data_ptr<float>() : nullptr,
                          running_var.has_value() ? running_var->data_ptr<float>() : nullptr, (float)eps,
                          (float)momentum, relu ? 1 : 0, cur_stream());
}

void bn_backward(const torch::Tensor& dy, const torch::Tensor& x, const torch::Tensor& y, torch::Tensor dx,
                 c10::optional<torch::Tensor> dres, const torch::Tensor& mean, const torch::Tensor& invstd,
                 const torch::Tensor& gamma, torch::Tensor acc, torch::Tensor dgamma, torch::Tensor dbeta, bool relu) {
  check_nhwc_bf16(dy, "dy");
  check_nhwc_bf16(x, "x");
  check_nhwc_bf16(dx, "dx");
  c10::cuda::CUDAGuard guard(x.device());
  const long long R = x.numel() / x.size(1);
  auto part = torch::empty({atomo_bn_partial_floats(R, (int)x.size(1))}, acc.options());
  atomo_launch_bn_backward(dy.data_ptr(), x.data_ptr(), y.data_ptr(), dx.data_ptr(),
                           dres.has_value() ? dres->data_ptr() : nullptr, R, (int)x.size(1), mean.data_ptr<float>(),
                           invstd.data_ptr<float>(), gamma.data_ptr<float>(), acc.data_ptr<float>(),
                           part.data_ptr<float>(), dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), relu ? 1 : 0,
                           cur_stream());
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
                uint64_t ctrl, uint64_t group_counter, int flags, uint64_t tstats, bool final_group, bool timed) {
  atomo_v2_launch_project(P<const void>(units), P<const void>(tiles), tile0, ntiles, P<const long long>(gptr),
                          P<const float>(vsel), P<const int>(selcount), P<float* const>(arena_peer),
                          P<int* const>(sig_peer), n_owners, arena_floats, worker, group, P<void>(ctrl),
                          P<unsigned int>(group_counter), flags, P<long long>(tstats), final_group ? 1 : 0,
                          timed ? 1 : 0, cur_stream());
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
void v2_wait_params(uint64_t sig, int n_owners, uint64_t ctrl, int64_t timeout, uint64_t tstats) {
  atomo_v2_launch_wait_params(P<const int>(sig), n_owners, P<void>(ctrl), timeout, P<long long>(tstats), cur_stream());
}
void v2_advance_step(uint64_t ctrl) { atomo_v2_launch_advance_step(P<void>(ctrl), cur_stream()); }
void v2_bcast_bytes(uint64_t src, uint64_t peer, uint64_t mc, int nranks, int self, int64_t nbytes) {
  atomo_v2_launch_bcast_bytes(P<const void>(src), P<void* const>(peer), P<void>(mc), nranks, self, nbytes,
                              cur_stream());
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
  m.def("v2_project", &v2_project);
  m.def("v2_ps", &v2_ps);
  m.def("v2_wait_params", &v2_wait_params);
  m.def("v2_advance_step", &v2_advance_step);
  m.def("v2_bcast_bytes", &v2_bcast_bytes);
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
