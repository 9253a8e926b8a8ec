// Kernel table of one env model: the rollout and step kernels built for it.  Each kernels_<model>.cu (one translation
// unit per model, compiled in parallel) instantiates model_kernels<Model, families>(); the host code looks the table
// up through kernels_of(model).
#pragma once
#include "kernel.cuh"
#include "rollout_tc2.cuh"

namespace gops {

struct LwArgs;
typedef void (*RolloutFn)(const KParams);
typedef void (*StepFn)(const KParams, const float*, int, float*, float*, float*);
typedef void (*LwFn)(const KParams, const LwArgs);

struct LwKernels {      // layer-wise path of the wide nets (lw_rollout.cuh)
  LwFn init, step, reverse;
};

struct ModelKernels {
  RolloutFn mma[2][3][4];   // fused mma.sync rollout [hidden 64 / 256][config (hidden 256: 0 only)][alg]
  RolloutFn tc[3][4];       // fused wgmma rollout [TcVariant][alg]; kTcGeluChain: FHADP only, one output
  LwKernels lw;
  StepFn step;              // gops_b200_model_step of the state == obs models
};

// families of a model beyond the fused mma.sync rollout
enum : unsigned { kWgmmaRollout = 1, kModelStep = 2 };

// Instantiations of the wgmma rollout: hidden activation and wrapper flags read at run time; GELU fixed at compile time;
// GELU, one action and the wrapper chain kTcChain fixed at compile time (FHADP of the models with one action only).
// kTcChain is what create_env_model builds by default on a model with unbounded observations (idpendulum): ScaleAction
// + ClipAction, no ScaleObservation, no ActionRepeat, no effective ClipObservation.
enum TcVariant { kTcGeneric = 0, kTcGelu = 1, kTcGeluChain = 2 };
constexpr unsigned kTcChain = kWrapActionScale | kWrapClipAction;

static_assert(ALG_FHADP == 0 && ALG_PIM == 1 && ALG_PEV == 2 && ALG_TRACE == 3, "table index = alg");

template <class M, int HD, int S, int NT>
void set_mma(RolloutFn (&fn)[4]) {
  fn[ALG_FHADP] = rollout_kernel<M, HD, S, NT, ALG_FHADP>;
  fn[ALG_PIM] = rollout_kernel<M, HD, S, NT, ALG_PIM>;
  fn[ALG_PEV] = rollout_kernel<M, HD, S, NT, ALG_PEV>;
  fn[ALG_TRACE] = rollout_kernel<M, HD, S, NT, ALG_TRACE>;
}

template <class M, int AF, int NA, class W>   // AF, NA, W: see rollout_tc2_kernel
void set_tc(RolloutFn (&fn)[4]) {
  fn[ALG_FHADP] = rollout_tc2_kernel<M, ALG_FHADP, AF, NA, W>;
  fn[ALG_PIM] = rollout_tc2_kernel<M, ALG_PIM, AF, NA, W>;
  fn[ALG_PEV] = rollout_tc2_kernel<M, ALG_PEV, AF, NA, W>;
  fn[ALG_TRACE] = rollout_tc2_kernel<M, ALG_TRACE, AF, NA, W>;
}

// The layer-wise kernels are passed in by the models that have them, so that lw_rollout.cuh (and its kernels) is only
// compiled into their objects.  NA: 1 for a model with one action, else MAXA.  Only with NA = 1 is the kTcGeluChain
// FHADP rollout built, for nets with one output.  With MAXA outputs or with the wrapper flags read at run time, fixing
// NA makes ptxas spill more than the generic kernel does (CUDA 12.9), so those stay generic.  The INFADP kernels stay
// generic as well: built this way, their value-net weight gradient on idpendulum differs from the generic kernel's in
// the last bit of a few entries, which the FHADP kernel's results do not.
template <class M, unsigned FAMILIES, int NA = MAXA>
ModelKernels model_kernels(LwKernels lw = {}) {
  ModelKernels k = {};
  set_mma<M, 64, 128, 512>(k.mma[0][0]);   // kConfigs of gops_b200.cu: sub-tile S, threads
  set_mma<M, 64, 64, 256>(k.mma[0][1]);
  set_mma<M, 64, 32, 128>(k.mma[0][2]);
  set_mma<M, 256, 32, 256>(k.mma[1][0]);   // kWideConfig
  if constexpr ((FAMILIES & kWgmmaRollout) != 0) {
    set_tc<M, -1, MAXA, WrapRt>(k.tc[kTcGeneric]);
    set_tc<M, GOPS_ACT_GELU, MAXA, WrapRt>(k.tc[kTcGelu]);
    if constexpr (NA == 1) k.tc[kTcGeluChain][ALG_FHADP] = rollout_tc2_kernel<M, ALG_FHADP, GOPS_ACT_GELU, NA, WrapFixed<kTcChain>>;
  }
  if constexpr ((FAMILIES & kModelStep) != 0) k.step = model_step_kernel<M>;
  k.lw = lw;
  return k;
}

const ModelKernels& kernels_idp();
const ModelKernels& kernels_lq();
const ModelKernels& kernels_vehconti();
const ModelKernels& kernels_vehtrack();
const ModelKernels& kernels_mobilerobot();

// veh3dof_tracking_detour (lw_detour.cuh, kernels_vehtrack.cu): forward / reverse step kernels of the layer-wise path
// (init is the model's), the model step and the loss / constraint scalars
LwFn lw_fn_vehtrack_detour(int which);   // 1 forward step, 2 reverse step
void launch_veh_step_detour(const KParams& p, const float* action, float* next_obs, float* reward, float* next_done,
                            float* next_state, cudaStream_t st);
void lw_launch_scalars_detour(const KParams& p, const float* vacc, const float* cacc, const float* dn_last, float* scalars,
                              cudaStream_t st);

}  // namespace gops
