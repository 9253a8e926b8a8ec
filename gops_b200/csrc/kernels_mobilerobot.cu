// Kernel table of ModelMobileRobot (own translation unit: parallel build).  No wgmma family: every rollout of this model
// runs on the fused mma.sync kernel.
#include "model_kernels.cuh"

namespace gops {

const ModelKernels& kernels_mobilerobot() {
  static const ModelKernels k = model_kernels<ModelMobileRobot, kModelStep>();
  return k;
}

}  // namespace gops
