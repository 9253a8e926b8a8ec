// Instantiations of the fused rollout kernel for ModelIdp (own translation unit: parallel build).
#include "kernel.cuh"
#include "lw_rollout.cuh"
#include "rollout_tc2.cuh"

namespace gops {

typedef void (*RolloutFn)(const KParams);
typedef void (*StepFn)(const KParams, const float*, int, float*, float*, float*);

template <int ALG>
static RolloutFn pick(int hid, int cfg) {
  if (hid > 64) return rollout_kernel<ModelIdp, 256, 32, 256, ALG>;
  switch (cfg) {
    case 0: return rollout_kernel<ModelIdp, 64, 128, 512, ALG>;
    case 1: return rollout_kernel<ModelIdp, 64, 64, 256, ALG>;
    default: return rollout_kernel<ModelIdp, 64, 32, 128, ALG>;
  }
}

RolloutFn rollout_fn_idp(int hid, int cfg, int alg) {
  switch (alg) {
    case ALG_FHADP: return pick<ALG_FHADP>(hid, cfg);
    case ALG_PIM: return pick<ALG_PIM>(hid, cfg);
    case ALG_PEV: return pick<ALG_PEV>(hid, cfg);
    default: return pick<ALG_TRACE>(hid, cfg);
  }
}
RolloutFn rollout_fn_tc2_idp(int alg, int hact) {   // wgmma rollout kernel (rollout_tc2.cuh)
  if (hact == GOPS_ACT_GELU) {                       // activation fixed at compile time (rollout_tc2.cuh, GOPS_TC2_ACT_SWITCH)
    switch (alg) {
      case ALG_FHADP: return rollout_tc2_kernel<ModelIdp, ALG_FHADP, GOPS_ACT_GELU>;
      case ALG_PIM: return rollout_tc2_kernel<ModelIdp, ALG_PIM, GOPS_ACT_GELU>;
      case ALG_PEV: return rollout_tc2_kernel<ModelIdp, ALG_PEV, GOPS_ACT_GELU>;
      default: return rollout_tc2_kernel<ModelIdp, ALG_TRACE, GOPS_ACT_GELU>;
    }
  }
  switch (alg) {
    case ALG_FHADP: return rollout_tc2_kernel<ModelIdp, ALG_FHADP>;
    case ALG_PIM: return rollout_tc2_kernel<ModelIdp, ALG_PIM>;
    case ALG_PEV: return rollout_tc2_kernel<ModelIdp, ALG_PEV>;
    default: return rollout_tc2_kernel<ModelIdp, ALG_TRACE>;
  }
}

StepFn step_fn_idp() { return model_step_kernel<ModelIdp>; }

LwFn lw_fn_idp(int which) {   // layer-wise path of the wide nets: init / forward step / reverse step
  switch (which) {
    case 0: return lw_init_kernel<ModelIdp>;
    case 1: return lw_step_kernel<ModelIdp>;
    default: return lw_reverse_kernel<ModelIdp>;
  }
}

}  // namespace gops
