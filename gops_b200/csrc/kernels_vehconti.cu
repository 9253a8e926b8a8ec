// Kernel table of ModelVehConti (own translation unit: parallel build).
#include "model_kernels.cuh"

namespace gops {

const ModelKernels& kernels_vehconti() {
  static const ModelKernels k = model_kernels<ModelVehConti, 0>();
  return k;
}

}  // namespace gops
