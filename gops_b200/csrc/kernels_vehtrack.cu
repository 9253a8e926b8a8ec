// Kernel table of ModelVehTrack and the veh3dof_tracking_detour kernels (own translation unit: parallel build).
#include "lw_rollout.cuh"
#include "lw_detour.cuh"
#include "model_kernels.cuh"

namespace gops {

const ModelKernels& kernels_vehtrack() {
  static const ModelKernels k = model_kernels<ModelVehTrack, 0>(
      {lw_init_kernel<ModelVehTrack>, lw_step_kernel<ModelVehTrack>, lw_reverse_kernel<ModelVehTrack>});
  return k;
}

LwFn lw_fn_vehtrack_detour(int which) {   // veh3dof_tracking_detour: forward step / reverse step (init is shared)
  return which == 1 ? lw_step_detour_kernel : lw_reverse_detour_kernel;
}
void launch_veh_step_detour(const KParams& p, const float* action, float* next_obs, float* reward, float* next_done,
                            float* next_state, cudaStream_t st) {
  veh_step_detour_kernel<<<(unsigned)((p.batch + 127) / 128), 128, 0, st>>>(p, action, next_obs, reward, next_done, next_state);
}
void lw_launch_scalars_detour(const KParams& p, const float* vacc, const float* cacc, const float* dn_last, float* scalars,
                              cudaStream_t st) {
  lw_scalars_detour_kernel<<<1, 256, 0, st>>>(p, vacc, cacc, dn_last, scalars);
}

}  // namespace gops
