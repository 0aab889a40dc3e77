// Lion on the bf16 engine: the code-selected launch of the PS kernels' Lion instantiation (PsArgsLion,
// v2_ps_common.cuh).  It decodes and sums exactly as the plain launch, steps master / mom (vectors: vparams / vmom)
// by the Lion rule, broadcasts the new parameters and completes the group; the last group publishes them.
#include "v2_ps_common.cuh"

namespace atomo {
namespace v2 {

extern "C" {

void atomo_v2_launch_ps_spectral_lion(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_qsgd_lion(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_entry_lion(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_sign_lion(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_fp8_lion(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_hadamard_lion(const void* args, int grid, cudaStream_t stream);
void atomo_v2_launch_ps_powersgd_lion(const void* args, int grid, cudaStream_t stream);

// `ps` selects the PS kernel of the code (0 spectral / dense, 1 QSGD / TernGrad, 2 entry-wise / top-k, 3 sign, 4 fp8,
// 5 hadamard, 6 PowerSGD), as in v2_ps_layerwise / v2_ps_gather
void atomo_v2_launch_ps_lion(int ps, const void* units, const void* tiles, int tile0, int ntiles, int W, int nranks,
                             int group, int final_group, int owner, float* master, float* mom, float* vmom,
                             void* wshadow_mc, void* const* wshadow_peer, float* vparams_local, float* vparams_mc,
                             float* const* vparams_peer, const float* vgrads_mc, const float* const* vgrads_peer,
                             const void* const* stage_peer, const float* arenas, long long arena_floats, int* sig,
                             int* const* sig_peer, void* ctrl, unsigned int* group_counter, long long timeout,
                             long long* tstats, float inv_w, int grid, cudaStream_t stream) {
  PsArgsLion a;
  static_cast<PsArgs2&>(a) =
      ps_args(units, tiles, tile0, ntiles, W, nranks, group, final_group, owner, master, mom, nullptr, nullptr, vmom,
              nullptr, nullptr, wshadow_mc, wshadow_peer, vparams_local, vparams_mc, vparams_peer, vgrads_mc,
              vgrads_peer, stage_peer, arenas, arena_floats, sig, sig_peer, ctrl, group_counter, timeout, tstats,
              inv_w);
  switch (ps) {
    case 0: atomo_v2_launch_ps_spectral_lion(&a, grid, stream); break;
    case 1: atomo_v2_launch_ps_qsgd_lion(&a, grid, stream); break;
    case 2: atomo_v2_launch_ps_entry_lion(&a, grid, stream); break;
    case 3: atomo_v2_launch_ps_sign_lion(&a, grid, stream); break;
    case 4: atomo_v2_launch_ps_fp8_lion(&a, grid, stream); break;
    case 5: atomo_v2_launch_ps_hadamard_lion(&a, grid, stream); break;
    default: atomo_v2_launch_ps_powersgd_lion(&a, grid, stream); break;
  }
}

}  // extern "C"
}  // namespace v2
}  // namespace atomo
