// Kernel table of ModelIdp (own translation unit: parallel build).
#include "lw_rollout.cuh"
#include "model_kernels.cuh"

namespace gops {

const ModelKernels& kernels_idp() {
  static const ModelKernels k = model_kernels<ModelIdp, kWgmmaRollout | kModelStep, 1>(   // one action
      {lw_init_kernel<ModelIdp>, lw_step_kernel<ModelIdp>, lw_reverse_kernel<ModelIdp>});
  return k;
}

}  // namespace gops
