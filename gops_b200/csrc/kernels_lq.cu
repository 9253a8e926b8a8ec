// Kernel table of ModelLq (own translation unit: parallel build).
#include "lw_rollout.cuh"
#include "model_kernels.cuh"

namespace gops {

const ModelKernels& kernels_lq() {
  static const ModelKernels k = model_kernels<ModelLq, kWgmmaRollout | kModelStep>(
      {lw_init_kernel<ModelLq>, lw_step_kernel<ModelLq>, lw_reverse_kernel<ModelLq>});
  return k;
}

}  // namespace gops
