// libgops_b200.so: C ABI (include/gops_b200.h) over the fused sm_90a rollout kernels.
#include "gops_b200.h"

#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <new>
#include <string>
#include <vector>

#include "kernel.cuh"
#include "aux_kernels.cuh"
#include "mlp_tc.cuh"
#include "rollout_tc2.cuh"
#include "lw_rollout.cuh"
#include <cuda_bf16.h>

using namespace gops;

namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};     // kernels launched by this library (gops_b200_launch_count)

int fail(const std::string& msg) {
  g_err = msg;
  return 1;
}
#define CUDA_OK(expr)                                                                          \
  do {                                                                                         \
    cudaError_t e__ = (expr);                                                                  \
    if (e__ != cudaSuccess)                                                                    \
      return fail(std::string(#expr) + ": " + cudaGetErrorString(e__));                        \
  } while (0)

#define CUDA_OK_L(expr, label)                                                                 \
  do {                                                                                         \
    cudaError_t e__ = (expr);                                                                  \
    if (e__ != cudaSuccess)                                                                    \
      return fail(std::string(label) + " " + #expr + ": " + cudaGetErrorString(e__));          \
  } while (0)

// A CUDA error left behind by an earlier (possibly foreign) call must not be blamed on the next launch.
#define ENTRY(name)                                                                            \
  do {                                                                                         \
    cudaError_t e0__ = cudaGetLastError();                                                     \
    if (e0__ != cudaSuccess && getenv("GOPS_B200_DEBUG"))                                      \
      fprintf(stderr, "[gops_b200] stale CUDA error at entry of %s: %s\n", name, cudaGetErrorString(e0__)); \
  } while (0)

int round4(int x) { return (x + 3) & ~3; }
}  // namespace
namespace gops {   // shared with the other translation units of the library (dense_tc.cu, dsac.cu)
int dense_fail(const std::string& msg) { return fail(msg); }
void dense_count_launch(int n) { g_launches += n; }
}  // namespace gops
namespace {

// Every entry point runs on the device that owns its plan / buffers, whatever the caller's current device is
// (networks on cuda:1 while cuda:0 is current must not put scratch on one GPU and the launch on the other).
struct DevGuard {
  int prev = -1;
  bool switched = false;
  explicit DevGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && dev >= 0 && prev != dev) switched = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DevGuard() {
    if (switched) cudaSetDevice(prev);
  }
};
int device_of(const void* p) {
  cudaPointerAttributes a;
  if (p && cudaPointerGetAttributes(&a, p) == cudaSuccess && a.type == cudaMemoryTypeDevice) return a.device;
  (void)cudaGetLastError();
  int d = 0;
  cudaGetDevice(&d);
  return d;
}
constexpr int kMaxDevices = 64;

bool make_net(const gops_b200_mlp_desc& d, NetL& L, std::string& why) {
  memset(&L, 0, sizeof(L));
  if (d.hidden != 64 && d.hidden != 256) {
    why = "hidden width " + std::to_string(d.hidden) + " not built (supported: 64, 256)";
    return false;
  }
  const int HID = d.hidden, HP = HID == 64 ? 72 : HID + 4;
  if (d.out_dim < 1 || d.out_dim > MAXA) { why = "out_dim out of range"; return false; }
  if (d.out_act != GOPS_ACT_LINEAR) { why = "output_activation other than 'linear' is not supported"; return false; }
  if (d.hidden_act < 0 || d.hidden_act > GOPS_ACT_LINEAR) { why = "bad hidden activation"; return false; }
  L.obs = d.in_dim;
  L.time_input = d.time_input ? 1 : 0;
  L.in = d.in_dim + L.time_input;
  L.in8 = (L.in + 7) & ~7;
  L.inp = L.in8;      // rows of the observation tile (pad rows stay zero)
  L.out = d.out_dim;
  L.hact = d.hidden_act;
  L.oact = d.out_act;
  int o = 0;
  if (HID == 64) {
    L.o_w1 = o; o += L.in8 * HP;
    L.o_w1l = o; o += L.in8 * HP;
    L.o_w2 = o; o += HID * HP;
    L.o_w2l = o; o += HID * HP;
  } else {
    L.o_w1 = o; o += L.in * HP;
    L.o_w2 = o; o += HID * HP;
    L.o_w1l = L.o_w1; L.o_w2l = L.o_w2;
  }
  L.o_w3 = o; o += round4(L.out * HID);
  L.o_b1 = o; o += HID;
  L.o_b2 = o; o += HID;
  L.o_b3 = o; o += 4;
  L.blob = o;
  int g = 0;
  L.g_w1 = g; g += HID * L.in;
  L.g_b1 = g; g += HID;
  L.g_w2 = g; g += HID * HID;
  L.g_b2 = g; g += HID;
  L.g_w3 = g; g += L.out * HID;
  L.g_b3 = g; g += L.out;
  L.nparam = g;
  // shared-memory accumulator layout (64-wide tensor-core path pads W2 rows to 68 floats; wide nets accumulate in
  // the global partial in torch layout)
  L.ldw2 = HID == 64 ? 68 : HID;
  int a = 0;
  L.d_w1 = a; a += HID * L.in;
  L.d_b1 = a; a += HID;
  L.d_w2 = a; a += HID * L.ldw2;
  L.d_b2 = a; a += HID;
  L.d_w3 = a; a += L.out * HID;
  L.d_b3 = a; a += L.out;
  L.nacc = a;
  return true;
}

struct Config {
  int S, NT;
};
const Config kConfigs[] = {{128, 512}, {64, 256}, {32, 128}};   // sub-tile S, threads (= samples per chunk)

const Config kWideConfig = {32, 256};   // hidden 256: activations only in smem, 8 sub-tiles per chunk

typedef void (*RolloutFn)(const KParams);
typedef void (*StepFn)(const KParams, const float*, int, float*, float*, float*);

}  // namespace

// one translation unit per env model (kernels_<model>.cu), compiled in parallel
namespace gops {
RolloutFn rollout_fn_idp(int hid, int cfg, int alg);
RolloutFn rollout_fn_lq(int hid, int cfg, int alg);
RolloutFn rollout_fn_vehconti(int hid, int cfg, int alg);
RolloutFn rollout_fn_vehtrack(int hid, int cfg, int alg);
StepFn step_fn_idp();
StepFn step_fn_lq();
LwFn lw_fn_idp(int which);              // layer-wise path (wide nets): 0 init, 1 forward step, 2 reverse step
LwFn lw_fn_lq(int which);
LwFn lw_fn_vehtrack(int which);
LwFn lw_fn_vehtrack_detour(int which);    // veh3dof_tracking_detour: 1 forward step, 2 reverse step (lw_detour.cuh)
void launch_veh_step_detour(const KParams& p, const float* action, float* next_obs, float* reward, float* next_done,
                            float* next_state, cudaStream_t st);
void lw_launch_scalars_detour(const KParams& p, const float* vacc, const float* cacc, const float* dn_last, float* scalars,
                              cudaStream_t st);
RolloutFn rollout_fn_tc2_idp(int alg, int hact);  // wgmma rollout kernel (rollout_tc2.cuh)
RolloutFn rollout_fn_tc2_lq(int alg, int hact);
}  // namespace gops

namespace {

RolloutFn rollout_fn(int model, int hid, int cfg, int alg) {
  switch (model) {
    case GOPS_MODEL_IDPENDULUM: return rollout_fn_idp(hid, cfg, alg);
    case GOPS_MODEL_LQ: return rollout_fn_lq(hid, cfg, alg);
    case GOPS_MODEL_VEH3DOFCONTI: return rollout_fn_vehconti(hid, cfg, alg);
    case GOPS_MODEL_VEH3DOF_TRACKING: return rollout_fn_vehtrack(hid, cfg, alg);
    default: return nullptr;
  }
}
RolloutFn rollout_fn_tc2(int model, int alg, int hact = -1) {      // hact: the nets' common hidden activation, or -1
  switch (model) {
    case GOPS_MODEL_IDPENDULUM: return rollout_fn_tc2_idp(alg, hact);
    case GOPS_MODEL_LQ: return rollout_fn_tc2_lq(alg, hact);
    default: return nullptr;
  }
}

LwFn lw_fn(int model, int which) {
  switch (model) {
    case GOPS_MODEL_IDPENDULUM: return lw_fn_idp(which);
    case GOPS_MODEL_LQ: return lw_fn_lq(which);
    case GOPS_MODEL_VEH3DOF_TRACKING: return lw_fn_vehtrack(which);
    default: return nullptr;
  }
}
StepFn step_fn(int model) {
  switch (model) {
    case GOPS_MODEL_IDPENDULUM: return step_fn_idp();
    case GOPS_MODEL_LQ: return step_fn_lq();
    default: return nullptr;
  }
}
int model_ns(int model) { return model == GOPS_MODEL_LQ ? LQN : (model == GOPS_MODEL_VEH3DOFCONTI ? 7 : 6); }

}  // namespace

struct gops_b200_plan {
  gops_b200_plan_desc desc;
  KParams kp;
  int device = 0, sm_count = 0, max_smem = 0;
  float *blob_pol = nullptr, *blob_val = nullptr, *blob_vtg = nullptr, *gpow = nullptr;
  float* tape = nullptr;
  size_t tape_floats = 0;
  float* partial = nullptr;
  size_t partial_floats = 0;
  float* ext_ref = nullptr;
  size_t ext_ref_floats = 0;
  float* xbuf = nullptr;
  size_t xbuf_floats = 0;
  float* blob_tc = nullptr;     // wgmma inference path: chunk-major hi / lo weight planes
  int blob_tc_floats = 0;
  // wgmma rollout kernel (BF16x3): NetL with the bf16-plane blob offsets, packed blobs
  bool tc_ok = false;
  NetL pol_tcf, val_tcf;
  int w_floats_tcf = 0;
  float *blob_pol_tcf = nullptr, *blob_val_tcf = nullptr, *blob_vtg_tcf = nullptr;
  bool tc2_attr_set[4] = {};
  float* osc = nullptr;   // obs scale | shift, 2 * obs_dim floats
  bool attr_set[4][4] = {};   // [alg][cfg]
  bool timing = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int path = GOPS_PATH_AUTO, last_path = 0;
  // layer-wise wgmma path of the wide nets (lw_rollout.cuh + dense_tc.cu)
  gops_b200_mlpnet* lw_net = nullptr;
  long long lw_cap = 0;
  float *lw_S = nullptr, *lw_Dn = nullptr, *lw_X = nullptr, *lw_Z = nullptr, *lw_Zb = nullptr, *lw_lam = nullptr,
        *lw_vacc = nullptr, *lw_dX = nullptr, *lw_sp = nullptr, *lw_cacc = nullptr, *lw_xcar = nullptr;
  std::vector<unsigned char> lw_key;      // the call the captured graph belongs to (KParams bytes + buffers + stream)
  int lw_key_hits = 0;
  cudaGraphExec_t lw_exec = nullptr;
  bool lw_graph_off = false;              // a capture attempt failed: this plan launches eagerly from then on
  cudaStream_t lw_cap_stream = nullptr;
  long long lw_graph_launches = 0;
  int last_grid = 0, last_S = 0, last_NT = 0;
  size_t last_smem = 0;
};

namespace {

size_t rollout_smem_bytes(const KParams& kp, int S, int NT) {
  const int SP = S + 4, XS = NT + 4, HID = kp.hid;
  // wide nets: + staging region R = max(obs sub-tile + 2 forward k-slices, 2 column slices)
  const size_t stage = (size_t)kp.inp_max * SP + 2 * 16 * (HID + 4);
  const size_t stage2 = 2 * (size_t)HID * 20;
  if (HID > 64) return sizeof(float) * (size_t)(4 + 4 * HID * SP + 8 * XS + (stage > stage2 ? stage : stage2));
  return sizeof(float) * (size_t)(4 + kp.w_floats + kp.dw_floats + kp.inp_max * XS + 4 * HID * SP + 8 * XS);
}
size_t infer_smem_bytes(const KParams& kp, int S, int NT) {
  const int SP = S + 4, XS = NT + 4, HID = kp.hid;
  if (HID > 64) return sizeof(float) * (size_t)(4 + 2 * HID * SP + 8 * XS + (size_t)kp.inp_max * SP + 2 * 16 * (HID + 4));
  return sizeof(float) * (size_t)(4 + kp.w_floats + kp.inp_max * XS + 2 * HID * SP + 8 * XS);
}

// NetL of the wgmma rollout path: blob = 3 bf16 planes of W1 ([2][64][8]) and W2 ([8][64][8]), then fp32 W3, b1, b2, b3
// (offsets in floats); shared-memory accumulators only for W3 / b3 (the rest is added into the FP32 partial every step)
void make_net_tcf(const NetL& base, NetL& L) {
  L = base;
  int o = 0;
  L.o_w1 = o; o += 3 * tcf::W1PLANE / 4;
  L.o_w1l = L.o_w1;
  L.o_w2 = o; o += 3 * tcf::W2PLANE / 4;
  L.o_w2l = L.o_w2;
  L.o_w3 = o; o += round4(L.out * 64);
  L.o_b1 = o; o += 64;
  L.o_b2 = o; o += 64;
  L.o_b3 = o; o += 4;
  L.blob = o;
  L.d_w3 = 0;
  L.d_b3 = L.out * 64;
  L.nacc = L.out * 64 + L.out;
}
// Path of a launch: the plan option (gops_b200_plan_set_path), overridden by GOPS_B200_ROLLOUT=tc|mma; AUTO takes the
// wgmma kernel wherever it is built for the plan (64-wide nets, <= 16 inputs, state == obs models)
bool rollout_use_tc(const gops_b200_plan* pl, long long batch) {
  if (!pl->tc_ok) return false;
  int path = pl->path;
  const char* e = getenv("GOPS_B200_ROLLOUT");
  if (e && !strcmp(e, "mma")) path = GOPS_PATH_MMA;
  if (e && !strcmp(e, "tc")) path = GOPS_PATH_TC;
  if (path == GOPS_PATH_MMA) return false;
  if (path == GOPS_PATH_TC) return true;
  // below ~2^14 samples the mma.sync kernel with its 32-sample tiles spreads the batch over more SMs and finishes
  // first.  Measured on one H100 80GB HBM3 (700 W) with the previous wgmma kernel (128-sample sub-tiles, one group per
  // SM), ms per update mma / wgmma: FHADP idpendulum H = 30  2^13 0.74 / 0.78, 2^14 1.20 / 0.78, 2^18 11.8 / 10.4;
  // INFADP lq s4a2 PEV + PIM  2^12 0.66 / 0.69, 2^14 0.86 / 0.71.  The current kernel (64-sample sub-tiles, three per
  // SM) is faster at 2^18; its crossover has not been re-measured.
  return batch >= 16384;
}
__global__ void pack_params_tcf_kernel(const float* __restrict__ flat, NetL L, float* __restrict__ blob) {
  const int n = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  __nv_bfloat16* w1 = reinterpret_cast<__nv_bfloat16*>(blob + L.o_w1);
  __nv_bfloat16* w2 = reinterpret_cast<__nv_bfloat16*>(blob + L.o_w2);
  auto put3 = [](float w, __nv_bfloat16* dst, int stride) {
    const __nv_bfloat16 b0 = __float2bfloat16_rn(w);
    const float r1 = w - __bfloat162float(b0);
    const __nv_bfloat16 b1 = __float2bfloat16_rn(r1);
    const float r2 = r1 - __bfloat162float(b1);
    dst[0] = b0; dst[stride] = b1; dst[2 * stride] = __float2bfloat16_rn(r2);
  };
  for (int i = t0; i < 2 * 64 * 8; i += n) {        // plane[kc][row n][8]: W1[n][8 kc + e]
    const int kc = i / 512, o = (i >> 3) & 63, k = 8 * kc + (i & 7);
    put3(k < L.in ? flat[L.g_w1 + o * L.in + k] : 0.f, w1 + i, 2 * 64 * 8);
  }
  for (int i = t0; i < 8 * 64 * 8; i += n) {
    const int kc = i / 512, o = (i >> 3) & 63, k = 8 * kc + (i & 7);
    put3(flat[L.g_w2 + o * 64 + k], w2 + i, 8 * 64 * 8);
  }
  for (int i = t0; i < L.out * 64; i += n) blob[L.o_w3 + i] = flat[L.g_w3 + i];
  for (int i = t0; i < 64; i += n) {
    blob[L.o_b1 + i] = flat[L.g_b1 + i];
    blob[L.o_b2 + i] = flat[L.g_b2 + i];
  }
  for (int i = t0; i < 4; i += n) blob[L.o_b3 + i] = i < L.out ? flat[L.g_b3 + i] : 0.f;
}
int launch_pack_tcf(const float* flat, const NetL& L, float* blob, cudaStream_t st) {
  pack_params_tcf_kernel<<<8, 256, 0, st>>>(flat, L, blob);
  ++g_launches;
  CUDA_OK_L(cudaGetLastError(), "launch#tcf-pack");
  return 0;
}

Config config_of(const gops_b200_plan* pl, int cfg) { return pl->kp.hid > 64 ? kWideConfig : kConfigs[cfg]; }

int pick_config(const gops_b200_plan* pl, long long B, bool infer) {
  if (pl->kp.hid > 64) return 0;
  // the largest chunk (threads per CTA) that still gives every SM at least one CTA
  const char* force = getenv("GOPS_B200_CFG");
  auto fits = [&](int c) {
    const size_t sm = infer ? infer_smem_bytes(pl->kp, kConfigs[c].S, kConfigs[c].NT)
                            : rollout_smem_bytes(pl->kp, kConfigs[c].S, kConfigs[c].NT);
    return sm <= (size_t)pl->max_smem;
  };
  if (force && force[0] >= '0' && force[0] <= '2' && fits(force[0] - '0')) return force[0] - '0';
  int best = -1;
  for (int c = 0; c < 3; ++c) {
    if (!fits(c)) continue;
    best = c;
    if (B >= (long long)pl->sm_count * kConfigs[c].NT) return c;
  }
  return best;
}

int ensure_scratch(gops_b200_plan* pl, int grid, int NT, int H, int part_rows_per_cta = 1) {
  const size_t need_tape = (size_t)grid * H * pl->kp.tape_ch * NT;
  if (need_tape > pl->tape_floats) {
    if (pl->tape) cudaFree(pl->tape);
    pl->tape = nullptr;
    CUDA_OK(cudaMalloc(&pl->tape, need_tape * sizeof(float)));
    pl->tape_floats = need_tape;
  }
  if (pl->desc.model == GOPS_MODEL_VEH3DOFCONTI) {
    const size_t need = (size_t)grid * (pl->kp.veh_P + 1 + H) * 4 * NT;
    if (need > pl->ext_ref_floats) {
      if (pl->ext_ref) cudaFree(pl->ext_ref);
      pl->ext_ref = nullptr;
      CUDA_OK(cudaMalloc(&pl->ext_ref, need * sizeof(float)));
      CUDA_OK(cudaMemset(pl->ext_ref, 0, need * sizeof(float)));
      pl->ext_ref_floats = need;
    }
  }
  if (pl->kp.hid > 64) {
    const size_t need = (size_t)grid * pl->kp.inp_max * (NT + 4);
    if (need > pl->xbuf_floats) {
      if (pl->xbuf) cudaFree(pl->xbuf);
      pl->xbuf = nullptr;
      CUDA_OK(cudaMalloc(&pl->xbuf, need * sizeof(float)));
      CUDA_OK(cudaMemset(pl->xbuf, 0, need * sizeof(float)));
      pl->xbuf_floats = need;
    }
  }
  const size_t need_part = (size_t)grid * part_rows_per_cta * pl->kp.part_stride;
  if (need_part > pl->partial_floats) {
    if (pl->partial) cudaFree(pl->partial);
    pl->partial = nullptr;
    CUDA_OK(cudaMalloc(&pl->partial, need_part * sizeof(float)));
    pl->partial_floats = need_part;
  }
  return 0;
}

int launch_pack(const float* flat, const NetL& L, int hid, float* blob, cudaStream_t st) {
  pack_params_kernel<<<hid > 64 ? 64 : 8, 256, 0, st>>>(flat, L, hid, blob);
  ++g_launches;
  CUDA_OK_L(cudaGetLastError(), "launch#1");
  return 0;
}

// Wide nets (hidden 256), FHADP: the layer-wise wgmma path.  AUTO takes it wherever it is built; MMA keeps the fused
// FP32-FFMA kernel (A/B baseline).
bool rollout_use_layerwise(const gops_b200_plan* pl, int alg) {
  if (pl->desc.open_loop || pl->desc.veh_detour) return alg == ALG_FHADP;
  if (pl->kp.hid <= 64 || alg != ALG_FHADP || pl->kp.horizon > 128) return false;
  if (!lw_fn(pl->desc.model, 0)) return false;
  int path = pl->path;
  const char* e = getenv("GOPS_B200_ROLLOUT");
  if (e && !strcmp(e, "mma")) path = GOPS_PATH_MMA;
  if (e && !strcmp(e, "tc")) path = GOPS_PATH_TC;
  return path != GOPS_PATH_MMA;
}

int launch_rollout_layerwise(gops_b200_plan* pl, const gops_b200_batch* b, const float* policy_params, cudaStream_t st,
                             float* grad_out, float* scalars_out) {
  KParams& kp = pl->kp;
  const int H = kp.horizon, A = kp.pol.out, in = kp.pol.in, ldx = round4(in), NS = model_ns(pl->desc.model);
  const long long B = b->batch;
  const bool open = pl->desc.open_loop != 0;
  if (open) {       // FHADP2: one policy evaluation emits all H actions; the rollout kernels read them strided
    if (B > pl->lw_cap || !pl->lw_net) {
      if (pl->lw_net) gops_b200_mlpnet_destroy(pl->lw_net);
      pl->lw_net = nullptr;
      float** bufs[] = {&pl->lw_S, &pl->lw_Dn, &pl->lw_Z, &pl->lw_Zb, &pl->lw_lam, &pl->lw_vacc, &pl->lw_sp};
      for (float** q : bufs) { cudaFree(*q); *q = nullptr; }
      const long long cap = (B + 127) / 128 * 128;
      const int32_t sizes[4] = {in, pl->desc.policy.hidden, pl->desc.policy.hidden, A * H};
      if (gops_b200_mlpnet_create(sizes, 4, kp.pol.hact, cap, 1, &pl->lw_net)) return 1;
      CUDA_OK(cudaMalloc(&pl->lw_S, sizeof(float) * (size_t)(H + 1) * NS * cap));
      CUDA_OK(cudaMalloc(&pl->lw_Dn, sizeof(float) * (size_t)(H + 1) * cap));
      CUDA_OK(cudaMalloc(&pl->lw_Z, sizeof(float) * (size_t)H * cap * A));
      CUDA_OK(cudaMalloc(&pl->lw_Zb, sizeof(float) * (size_t)H * cap * A));
      CUDA_OK(cudaMalloc(&pl->lw_lam, sizeof(float) * (size_t)NS * cap));
      CUDA_OK(cudaMalloc(&pl->lw_vacc, sizeof(float) * (size_t)cap));
      CUDA_OK(cudaMalloc(&pl->lw_sp, sizeof(float) * 2 * 256));
      pl->lw_cap = cap;
    }
    kp.alg = ALG_FHADP;
    kp.batch = B;
    kp.obs = b->obs; kp.done = b->done; kp.state = b->state; kp.reference = b->reference;
    kp.ref_t = b->ref_t; kp.ref_len = b->ref_len;
    LwFn f_init = lw_fn(pl->desc.model, 0), f_step = lw_fn(pl->desc.model, 1), f_rev = lw_fn(pl->desc.model, 2);
    LwArgs a;
    memset(&a, 0, sizeof(a));
    a.ldx = ldx; a.act_dim = A; a.bstride = pl->lw_cap; a.zs_k = A; a.zs_b = (long long)H * A;
    a.S = pl->lw_S; a.Dn = pl->lw_Dn; a.X = nullptr; a.Z = pl->lw_Z; a.Zb = pl->lw_Zb; a.lam = pl->lw_lam; a.vacc = pl->lw_vacc;
    const unsigned grid = (unsigned)((B + 127) / 128);
    if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev0, st));
    if (gops_b200_mlpnet_pack(pl->lw_net, policy_params, st)) return 1;
    if (gops_b200_mlpnet_forward(pl->lw_net, b->obs, kp.pol.obs, B, 0, 1, pl->lw_Z, H * A, st)) return 1;
    f_init<<<grid, 128, 0, st>>>(kp, a);
    const int sub = pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING ? LW_SUB : 1;
    const unsigned grid_step = (unsigned)((B * sub + 127) / 128);
    for (int k = 0; k < H; ++k) {
      a.k = k;
      f_step<<<grid_step, 128, 0, st>>>(kp, a);
    }
    for (int k = H - 1; k >= 0; --k) {
      a.k = k;
      f_rev<<<grid, 128, 0, st>>>(kp, a);
    }
    g_launches += 1 + 2 * H;
    if (gops_b200_mlpnet_backward(pl->lw_net, pl->lw_Zb, H * A, B, 0, grad_out, 0, nullptr, 0, st)) return 1;
    const int nb = 64;
    lw_scalars_kernel<<<nb, 256, 0, st>>>(pl->lw_vacc, pl->lw_Dn + (size_t)H * B, B, kp.inv_B, pl->lw_sp);
    lw_scalars_final_kernel<<<1, 32, 0, st>>>(pl->lw_sp, nb, scalars_out);
    g_launches += 2;
    CUDA_OK_L(cudaGetLastError(), "open-loop rollout");
    if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev1, st));
    pl->last_grid = (int)grid; pl->last_S = 128; pl->last_NT = 128; pl->last_smem = 0; pl->last_path = GOPS_PATH_TC;
    return 0;
  }
  if (B > pl->lw_cap || !pl->lw_net) {
    if (pl->lw_net) gops_b200_mlpnet_destroy(pl->lw_net);
    pl->lw_net = nullptr;
    float** bufs[] = {&pl->lw_S, &pl->lw_Dn, &pl->lw_X, &pl->lw_Z, &pl->lw_Zb, &pl->lw_lam, &pl->lw_vacc, &pl->lw_dX, &pl->lw_sp,
                      &pl->lw_cacc, &pl->lw_xcar};
    for (float** q : bufs) { cudaFree(*q); *q = nullptr; }
    const long long cap = (B + 127) / 128 * 128;
    const int32_t sizes[4] = {in, kp.hid, kp.hid, A};
    if (pl->lw_exec) { cudaGraphExecDestroy(pl->lw_exec); pl->lw_exec = nullptr; }
    pl->lw_key.clear();
    if (gops_b200_mlpnet_create(sizes, 4, kp.pol.hact, cap, H, &pl->lw_net)) return 1;
    if (gops_b200_mlpnet_keep_deltas(pl->lw_net, 1)) return 1;
    CUDA_OK(cudaMalloc(&pl->lw_S, sizeof(float) * (size_t)(H + 1) * NS * cap));
    CUDA_OK(cudaMalloc(&pl->lw_Dn, sizeof(float) * (size_t)(H + 1) * cap));
    CUDA_OK(cudaMalloc(&pl->lw_X, sizeof(float) * (size_t)(H + 1) * cap * ldx));
    CUDA_OK(cudaMalloc(&pl->lw_Z, sizeof(float) * (size_t)H * cap * A));
    CUDA_OK(cudaMalloc(&pl->lw_Zb, sizeof(float) * (size_t)H * cap * A));
    CUDA_OK(cudaMalloc(&pl->lw_lam, sizeof(float) * (size_t)NS * cap));
    CUDA_OK(cudaMalloc(&pl->lw_vacc, sizeof(float) * (size_t)cap));
    CUDA_OK(cudaMalloc(&pl->lw_dX, sizeof(float) * (size_t)cap * ldx));
    CUDA_OK(cudaMalloc(&pl->lw_sp, sizeof(float) * 2 * 256));
    if (pl->desc.veh_detour) {
      CUDA_OK(cudaMalloc(&pl->lw_cacc, sizeof(float) * 3 * (size_t)cap));
      CUDA_OK(cudaMalloc(&pl->lw_xcar, sizeof(float) * (size_t)cap * ldx));
    }
    pl->lw_cap = cap;
  }
  const long long cap = pl->lw_cap;
  kp.alg = ALG_FHADP;
  kp.batch = B;
  kp.obs = b->obs; kp.done = b->done; kp.state = b->state; kp.reference = b->reference;
  kp.ref_t = b->ref_t; kp.ref_len = b->ref_len;
  kp.surr = b->surr; kp.surr_len = b->surr_len;
  const bool detour = pl->desc.veh_detour != 0;
  LwFn f_init = lw_fn(pl->desc.model, 0), f_step = detour ? lw_fn_vehtrack_detour(1) : lw_fn(pl->desc.model, 1),
       f_rev = detour ? lw_fn_vehtrack_detour(2) : lw_fn(pl->desc.model, 2);
  LwArgs a;
  memset(&a, 0, sizeof(a));
  a.cacc = pl->lw_cacc; a.xcar = pl->lw_xcar;
  a.ldx = ldx; a.act_dim = A; a.bstride = cap; a.zs_k = cap * A; a.zs_b = A;
  a.S = pl->lw_S; a.Dn = pl->lw_Dn; a.X = pl->lw_X; a.Z = pl->lw_Z; a.Zb = pl->lw_Zb; a.lam = pl->lw_lam; a.vacc = pl->lw_vacc;
  // S / Dn are indexed with the real batch as the row count
  const unsigned grid = (unsigned)((B + 127) / 128);
  if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev0, st));
  // The update is ~10 launches per horizon step, each a few microseconds: once the same call (same buffers, same
  // constants) has been seen twice it is captured into a CUDA graph and replayed, which removes the launch gaps.
  auto enqueue = [&](cudaStream_t st) -> int {
  if (gops_b200_mlpnet_pack(pl->lw_net, policy_params, st)) return 1;
  f_init<<<grid, 128, 0, st>>>(kp, a);
  ++g_launches;
  if (detour) {
    CUDA_OK(cudaMemsetAsync(pl->lw_cacc, 0, sizeof(float) * 3 * (size_t)B, st));
    CUDA_OK(cudaMemsetAsync(pl->lw_xcar, 0, sizeof(float) * (size_t)B * ldx, st));
  }
  const int sub = pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING ? LW_SUB : 1;
  const unsigned grid_step = (unsigned)((B * sub + 127) / 128);
  for (int k = 0; k < H; ++k) {
    if (gops_b200_mlpnet_forward(pl->lw_net, pl->lw_X + (size_t)k * cap * ldx, ldx, B, k, 1, pl->lw_Z + (size_t)k * cap * A, A, st))
      return 1;
    a.k = k;
    f_step<<<grid_step, 128, 0, st>>>(kp, a);
    ++g_launches;
  }
  for (int k = H - 1; k >= 0; --k) {
    a.k = k;
    a.dX = k == H - 1 ? nullptr : pl->lw_dX;
    f_rev<<<grid, 128, 0, st>>>(kp, a);
    ++g_launches;
    if (gops_b200_mlpnet_backward(pl->lw_net, pl->lw_Zb + (size_t)k * cap * A, A, B, k, nullptr, 0, k > 0 ? pl->lw_dX : nullptr, ldx,
                                  st))
      return 1;
  }
  if (gops_b200_mlpnet_wgrad_slots(pl->lw_net, 0, H, B, pl->lw_X, ldx, cap, pl->lw_Zb, A, cap, grad_out, 0, st)) return 1;
  const int nb = 64;
  if (detour) {
    lw_launch_scalars_detour(kp, pl->lw_vacc, pl->lw_cacc, pl->lw_Dn + (size_t)H * B, scalars_out, st);
    g_launches += 1;
  } else {
    lw_scalars_kernel<<<nb, 256, 0, st>>>(pl->lw_vacc, pl->lw_Dn + (size_t)H * B, B, kp.inv_B, pl->lw_sp);
    lw_scalars_final_kernel<<<1, 32, 0, st>>>(pl->lw_sp, nb, scalars_out);
    g_launches += 2;
  }
  CUDA_OK_L(cudaGetLastError(), "layer-wise rollout");
  return 0;
  };
  std::vector<unsigned char> key(sizeof(KParams) + 4 * sizeof(void*));
  memcpy(key.data(), &kp, sizeof(KParams));
  const void* kptr[4] = {policy_params, grad_out, scalars_out, (const void*)st};
  memcpy(key.data() + sizeof(KParams), kptr, sizeof(kptr));
  const char* ge = getenv("GOPS_B200_GRAPH");
  const bool graphs = !(ge && !strcmp(ge, "0"));
  if (pl->lw_exec && key == pl->lw_key) {
    CUDA_OK(cudaGraphLaunch(pl->lw_exec, st));
    g_launches += pl->lw_graph_launches;
  } else {
    if (key == pl->lw_key) ++pl->lw_key_hits;
    else {
      pl->lw_key = key;
      pl->lw_key_hits = 0;
      if (pl->lw_exec) { cudaGraphExecDestroy(pl->lw_exec); pl->lw_exec = nullptr; }
    }
    bool replayed = false;
    if (graphs && !pl->lw_graph_off && pl->lw_key_hits >= 1) {
      const long long n0 = g_launches;
      // torch's default stream is the legacy stream, which cannot be captured: record on a private stream (nothing
      // executes during capture), replay on the caller's.  Capture is an optimisation only: if any step of it fails the
      // plan keeps launching eagerly (nothing has run yet at that point) and does not try again.
      bool ok = pl->lw_cap_stream != nullptr || cudaStreamCreateWithFlags(&pl->lw_cap_stream, cudaStreamNonBlocking) == cudaSuccess;
      ok = ok && cudaStreamBeginCapture(pl->lw_cap_stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
      if (ok) {
        const int rc = enqueue(pl->lw_cap_stream);
        cudaGraph_t g = nullptr;
        const cudaError_t ce = cudaStreamEndCapture(pl->lw_cap_stream, &g);
        ok = rc == 0 && ce == cudaSuccess && g != nullptr && cudaGraphInstantiate(&pl->lw_exec, g, 0) == cudaSuccess;
        if (g) cudaGraphDestroy(g);
      }
      if (ok) {
        pl->lw_graph_launches = g_launches - n0;
        CUDA_OK(cudaGraphLaunch(pl->lw_exec, st));
        replayed = true;
      } else {
        (void)cudaGetLastError();
        if (pl->lw_exec) { cudaGraphExecDestroy(pl->lw_exec); pl->lw_exec = nullptr; }
        pl->lw_graph_off = true;
        g_launches = n0;
      }
    }
    if (!replayed && enqueue(st)) return 1;
  }
  if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev1, st));
  pl->last_grid = (int)grid; pl->last_S = 128; pl->last_NT = 128; pl->last_smem = 0; pl->last_path = GOPS_PATH_TC;
  return 0;
}

int launch_rollout(gops_b200_plan* pl, const gops_b200_batch* b, int alg, cudaStream_t st, float* grad_out,
                   float* scalars_out) {
  if (!b || b->batch <= 0) return fail("empty batch");
  if (!b->obs || !b->done) return fail("obs/done pointers are required");
  if (pl->desc.model == GOPS_MODEL_VEH3DOFCONTI &&
      (!b->state || !b->ref_points || !b->path_num || !b->u_num || !b->ref_time))
    return fail("pyth_veh3dofconti needs state, ref_points, path_num, u_num, ref_time");
  if (pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING) {
    if (!b->state || !b->reference) return fail("veh3dof_tracking needs state (robot_state) and reference");
    if (b->ref_t < 0 || b->ref_t + pl->kp.horizon + pl->kp.veh_P + 1 > b->ref_len)
      return fail("veh3dof_tracking: reference too short for t + horizon + pre_horizon + 1 points");
  }
  KParams& kp = pl->kp;
  if (rollout_use_tc(pl, b->batch)) {
    const int hact = (alg == ALG_FHADP || pl->pol_tcf.hact == pl->val_tcf.hact) ? pl->pol_tcf.hact : -1;
    RolloutFn fn = rollout_fn_tc2(pl->desc.model, alg, hact);
    if (!fn) return fail("wgmma rollout kernel not built for this env model");
    const int S = tc2::GT, NT = tc2::NT2;
    KParams k2 = kp;
    k2.pol = pl->pol_tcf;
    k2.val = pl->val_tcf;
    k2.blob_pol = pl->blob_pol_tcf; k2.blob_val = pl->blob_val_tcf; k2.blob_vtg = pl->blob_vtg_tcf;
    k2.w_floats = pl->w_floats_tcf;
    k2.alg = alg;
    k2.batch = b->batch;
    k2.n_tiles = (int)((b->batch + NT - 1) / NT);
    k2.tape_ch = model_ns(pl->desc.model) + 1 + k2.pol.out;
    kp.tape_ch = k2.tape_ch;                        // ensure_scratch sizes the tape / partials from the plan's copy
    k2.obs = b->obs; k2.done = b->done; k2.state = b->state; k2.ref_points = b->ref_points;
    k2.path_num = b->path_num; k2.u_num = b->u_num; k2.ref_time = b->ref_time; k2.reference = b->reference;
    k2.ref_t = b->ref_t;
    k2.ref_len = b->ref_len;
    const NetL& upd = (alg == ALG_PEV) ? k2.val : k2.pol;
    k2.part_stride = round4(upd.nparam + 4);
    kp.part_stride = k2.part_stride;
    k2.dw_floats = round4(upd.nacc);
    const size_t smem = tc2::smem_bytes(k2.w_floats);
    if (smem > (size_t)pl->max_smem) return fail("wgmma rollout kernel does not fit in shared memory");
    bool& attr = pl->tc2_attr_set[alg];
    if (!attr) {
      CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, pl->max_smem));
      attr = true;
    }
    // one CTA per SM (shared memory); a batch of fewer sub-tiles than SMs gets one CTA per sub-tile, so that it spreads
    // over the SMs (the kernel leaves the other warpgroups of such a CTA idle)
    const long long subtiles = (b->batch + S - 1) / S;
    const int grid = (int)(subtiles < pl->sm_count ? subtiles : pl->sm_count);
    const int rows = tc2::WGS;                     // gradient partial rows (= independent warpgroups) per CTA
    if (ensure_scratch(pl, grid, tc2::WGS * tc2::GT, k2.horizon, rows)) return 1;   // tape columns per CTA
    k2.tape = pl->tape;
    k2.ext_ref = pl->ext_ref;
    k2.xbuf = pl->xbuf;
    k2.partial = pl->partial;
    if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev0, st));
    fn<<<grid, NT, smem, st>>>(k2);
    ++g_launches;
    CUDA_OK_L(cudaGetLastError(), "launch#2-tc");
    if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev1, st));
    pl->last_grid = grid; pl->last_S = S; pl->last_NT = NT; pl->last_smem = smem; pl->last_path = GOPS_PATH_TC;
    if (alg != ALG_TRACE) {
      const int n = upd.nparam + 4;
      reduce_partials_kernel<<<(n + 255) / 256, 256, 0, st>>>(pl->partial, grid * rows, k2.part_stride, upd.nparam, grad_out,
                                                             scalars_out);
      ++g_launches;
      CUDA_OK_L(cudaGetLastError(), "launch#3-tc");
    }
    return 0;
  }
  const int cfg = pick_config(pl, b->batch, false);
  if (cfg < 0) return fail("no kernel configuration fits in shared memory");
  const int S = config_of(pl, cfg).S, NT = config_of(pl, cfg).NT;
  RolloutFn fn = rollout_fn(pl->desc.model, kp.hid, cfg, alg);
  if (!fn) return fail("env model kind not built into this library");
  kp.alg = alg;
  kp.batch = b->batch;
  kp.n_tiles = (int)((b->batch + NT - 1) / NT);
  kp.tape_ch = model_ns(pl->desc.model) + 1 + kp.pol.out;
  kp.obs = b->obs; kp.done = b->done; kp.state = b->state; kp.ref_points = b->ref_points;
  kp.path_num = b->path_num; kp.u_num = b->u_num; kp.ref_time = b->ref_time; kp.reference = b->reference;
  kp.ref_t = b->ref_t;
  kp.ref_len = b->ref_len;
  const NetL& upd = (alg == ALG_PEV) ? kp.val : kp.pol;
  kp.part_stride = round4(upd.nparam + 4);
  kp.dw_floats = round4(upd.nacc);
  const size_t smem = rollout_smem_bytes(kp, S, NT);
  if (smem > (size_t)pl->max_smem) return fail("rollout kernel does not fit in shared memory");
  bool& attr = pl->attr_set[alg][cfg];
  if (!attr) {
    CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, pl->max_smem));
    attr = true;
  }
  int occ = 1;
  CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, NT, smem));
  if (occ < 1) return fail("rollout kernel does not fit on an SM");
  // one CTA per SM slot as long as every CTA still gets at least one S-sample sub-tile: the kernel splits the
  // batch into balanced contiguous ranges, so small batches spread over all SMs with partially filled chunks
  const long long slots = (long long)pl->sm_count * occ;
  const long long subtiles = (b->batch + S - 1) / S;
  const int grid = (int)(subtiles < slots ? subtiles : slots);
  if (ensure_scratch(pl, grid, NT, kp.horizon)) return 1;
  kp.tape = pl->tape;
  kp.ext_ref = pl->ext_ref;
  kp.xbuf = pl->xbuf;
  kp.partial = pl->partial;
  if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev0, st));
  fn<<<grid, NT, smem, st>>>(kp);
  ++g_launches;
  CUDA_OK_L(cudaGetLastError(), "launch#2");
  if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev1, st));
  pl->last_grid = grid; pl->last_S = S; pl->last_NT = NT; pl->last_smem = smem; pl->last_path = GOPS_PATH_MMA;
  if (alg != ALG_TRACE) {
    const int n = upd.nparam + 4;
    reduce_partials_kernel<<<(n + 255) / 256, 256, 0, st>>>(pl->partial, grid, kp.part_stride, upd.nparam, grad_out,
                                                           scalars_out);
    ++g_launches;
    CUDA_OK_L(cudaGetLastError(), "launch#3");
  }
  return 0;
}

}  // namespace

extern "C" {

int gops_b200_version(void) { return GOPS_B200_ABI_VERSION; }
int64_t gops_b200_launch_count(void) { return (int64_t)g_launches.load(); }
const char* gops_b200_last_error(void) { return g_err.c_str(); }

int gops_b200_plan_create(const gops_b200_plan_desc* d, gops_b200_plan** out) {
  ENTRY("gops_b200_plan_create(const gops_b200_pl");
  if (!d || !out) return fail("null argument");
  *out = nullptr;
  if (d->alg < GOPS_ALG_FHADP || d->alg > GOPS_ALG_INFADP_VALUE) return fail("unknown algorithm kind");
  if (d->horizon < 1 || d->horizon > 4096) return fail("horizon out of range");
  if (!rollout_fn(d->model, d->policy.hidden == 64 ? 64 : 256, 0, d->alg)) return fail("env model kind not built into this library");
  gops_b200_plan* pl = new (std::nothrow) gops_b200_plan();
  if (!pl) return fail("out of host memory");
  pl->desc = *d;
  KParams& kp = pl->kp;
  memset(&kp, 0, sizeof(kp));
  std::string why;
  gops_b200_mlp_desc pol_desc = d->policy;
  if (d->open_loop) {
    if (d->alg != GOPS_ALG_FHADP) { delete pl; return fail("open_loop (FHADP2) needs alg = GOPS_ALG_FHADP"); }
    if (d->policy.time_input || d->policy.out_dim % d->horizon || d->policy.out_dim > 256) {
      delete pl;
      return fail("open_loop: policy.out_dim must be act_dim * horizon (<= 256), without time input");
    }
    pol_desc.out_dim = d->policy.out_dim / d->horizon;      // kp.pol describes ONE step's action block
    if (pol_desc.hidden != 64 && pol_desc.hidden != 256) pol_desc.hidden = 256;   // geometry only; the mlpnet takes the real width
  }
  if (!make_net(pol_desc, kp.pol, why)) { delete pl; return fail("policy: " + why); }
  const bool infadp = d->alg != GOPS_ALG_FHADP;
  if (infadp) {
    if (!make_net(d->value, kp.val, why)) { delete pl; return fail("value: " + why); }
    if (d->value.out_dim != 1 || d->value.time_input) { delete pl; return fail("value net must be StateValue (out 1)"); }
    if (d->value.in_dim != d->policy.in_dim) { delete pl; return fail("value/policy obs dims differ"); }
  } else {
    kp.val = kp.pol;
  }
  const int act_dim = pol_desc.out_dim;
  int obs_dim_model = 0;
  if (d->model == GOPS_MODEL_IDPENDULUM) obs_dim_model = 6;
  if (d->model == GOPS_MODEL_LQ) {
    if (d->lq_n < 1 || d->lq_n > LQN || d->lq_m < 1 || d->lq_m > MAXA) { delete pl; return fail("lq dims out of range"); }
    obs_dim_model = d->lq_n;
    if (act_dim != d->lq_m) { delete pl; return fail("policy out_dim != lq action dim"); }
  }
  if (d->model == GOPS_MODEL_VEH3DOFCONTI || d->model == GOPS_MODEL_VEH3DOF_TRACKING) {
    if (d->veh_pre_horizon < 1) { delete pl; return fail("veh_pre_horizon must be >= 1"); }
    obs_dim_model = 6 + 4 * d->veh_pre_horizon + (d->veh_detour ? 4 : 0);
    if (act_dim != 2) { delete pl; return fail("vehicle models have 2 actions"); }
    if (d->veh_detour) {
      if (d->veh_detour != 1 && d->veh_detour != 2) { delete pl; return fail("veh_detour: 1 (detour) or 2 (surrcstr)"); }
      if (d->model != GOPS_MODEL_VEH3DOF_TRACKING || d->alg != GOPS_ALG_FHADP || d->open_loop) {
        delete pl;
        return fail("veh3dof_tracking_detour is built for FHADP and its constrained variants (closed-loop policy) only");
      }
      if (d->obs_scaling) { delete pl; return fail("veh3dof_tracking_detour: ScaleObservation is not built"); }
      if (!(d->veh_length > d->veh_width) || !(d->veh_width > 0.f)) { delete pl; return fail("veh3dof_tracking_detour: need veh_length > veh_width > 0"); }
    }
    if (d->clip_obs) {
      // the vehicle models declare +-inf observation bounds (pyth_veh3dofconti_model.py:79-88): identity clip
    }
  }
  if (d->policy.in_dim != obs_dim_model) { delete pl; return fail("policy in_dim does not match the env model obs_dim"); }
  if (d->model == GOPS_MODEL_IDPENDULUM && act_dim != 1) { delete pl; return fail("idpendulum has 1 action"); }

  kp.horizon = d->horizon;
  kp.hid = pol_desc.hidden;
  if (d->open_loop && !lw_fn(d->model, 0)) { delete pl; return fail("open_loop (FHADP2) is not built for this env model"); }
  if (infadp && d->value.hidden != d->policy.hidden) { delete pl; return fail("policy and value hidden widths differ"); }
  kp.gamma = d->gamma;
  kp.w_floats = kp.pol.blob > kp.val.blob ? kp.pol.blob : kp.val.blob;
  kp.inp_max = kp.pol.inp > kp.val.inp ? kp.pol.inp : kp.val.inp;
  kp.dw_floats = round4(kp.pol.nacc > kp.val.nacc ? kp.pol.nacc : kp.val.nacc);
  kp.action_scale = d->action_scale; kp.clip_action = d->clip_action; kp.mask_at_done = d->mask_at_done;
  kp.reward_shaping = d->reward_shaping; kp.reward_shift = d->reward_shift; kp.reward_scale = d->reward_scale;
  kp.obs_scaling = d->obs_scaling ? 1 : 0;
  kp.repeat_num = d->repeat_num > 0 ? d->repeat_num : 0;
  kp.sum_reward = d->sum_reward ? 1 : 0;
  if (kp.repeat_num > 0 && !(d->model == GOPS_MODEL_IDPENDULUM || d->model == GOPS_MODEL_LQ)) {
    delete pl;
    return fail("repeat_num (ActionRepeat) is supported for state==obs models only (not built for vehicle models)");
  }
  if (kp.repeat_num > 16) { delete pl; return fail("repeat_num > 16 not supported"); }
  if (kp.obs_scaling && (!d->obs_scale || !d->obs_shift)) { delete pl; return fail("obs_scaling without obs_scale/obs_shift arrays"); }
  bool finite_obs_bound = false;
  for (int j = 0; j < MAXA; ++j) {
    kp.min_action[j] = d->min_action[j]; kp.max_action[j] = d->max_action[j];
    kp.act_low[j] = d->act_low[j]; kp.act_high[j] = d->act_high[j];
    // (act_high_lim - act_low_lim) / 2 and (act_high_lim + act_low_lim) / 2 in fp32, mlp.py:74-76
    kp.pol_half[j] = (d->pol_act_high[j] - d->pol_act_low[j]) / 2.f;
    kp.pol_mid[j] = (d->pol_act_high[j] + d->pol_act_low[j]) / 2.f;
  }
  const bool state_is_obs = d->model == GOPS_MODEL_IDPENDULUM || d->model == GOPS_MODEL_LQ;
  for (int f = 0; f < LQN; ++f) {
    kp.obs_low[f] = (state_is_obs && f < obs_dim_model) ? d->obs_low[f] : -INFINITY;
    kp.obs_high[f] = (state_is_obs && f < obs_dim_model) ? d->obs_high[f] : INFINITY;
    if (isfinite(kp.obs_low[f]) || isfinite(kp.obs_high[f])) finite_obs_bound = true;
  }
  kp.clip_obs = (d->clip_obs && finite_obs_bound) ? 1 : 0;   // clipping to +-inf is the identity
  kp.lq_n = d->lq_n; kp.lq_m = d->lq_m; kp.lq_dt = d->lq_dt; kp.lq_rs = d->lq_reward_scale; kp.lq_rsh = d->lq_reward_shift;
  if (d->model == GOPS_MODEL_LQ) {
    for (int i = 0; i < d->lq_n; ++i) {
      for (int j = 0; j < d->lq_n; ++j) kp.lq_inv_IA[i * LQN + j] = d->lq_inv_IA[i * d->lq_n + j];
      for (int j = 0; j < d->lq_m; ++j) kp.lq_B[i * MAXA + j] = d->lq_B[i * d->lq_m + j];
      kp.lq_Q[i] = d->lq_Q[i];
    }
    for (int j = 0; j < d->lq_m; ++j) kp.lq_R[j] = d->lq_R[j];
  }
  {
    const gops_b200_reftraj& r = d->reftraj;
    RtC& q = kp.rt;
    q.sine_A = (float)r.sine_A; q.sine_omega = (float)r.sine_omega; q.sine_phi = (float)r.sine_phi;
    q.dl_t1 = (float)r.dl_t1; q.dl_t2 = (float)r.dl_t2; q.dl_t3 = (float)r.dl_t3; q.dl_t4 = (float)r.dl_t4;
    q.dl_y1 = (float)r.dl_y1; q.dl_y2 = (float)r.dl_y2;
    q.dl_k1 = (float)((r.dl_y2 - r.dl_y1) / (r.dl_t2 - r.dl_t1));
    q.dl_k2 = (float)((r.dl_y1 - r.dl_y2) / (r.dl_t4 - r.dl_t3));
    q.tri_k1 = (float)(2 * r.tri_A / r.tri_T); q.tri_k2 = (float)(-2 * r.tri_A / r.tri_T);
    q.tri_T = (float)r.tri_T; q.tri_half = (float)(r.tri_T / 2);
    q.circ_r = (float)r.circ_r;
    q.sp_A = (float)r.sp_A; q.sp_omega = (float)r.sp_omega; q.sp_phi = (float)r.sp_phi; q.sp_b = (float)r.sp_b;
    q.sp_c1 = (float)(-r.sp_A / r.sp_omega); q.sp_c3 = (float)(r.sp_A / r.sp_omega * cos(r.sp_phi));
    q.sp_const = (float)r.sp_const;
  }
  kp.cstr_mode = 0; kp.cstr_coef = 1.f;
  kp.cstr_y_tol = d->veh_y_error_tol; kp.cstr_u_tol = d->veh_u_error_tol;
  kp.veh_P = d->veh_pre_horizon;
  kp.veh_detour = d->veh_detour ? 1 : 0;
  kp.veh_dc = (float)(((double)d->veh_length - (double)d->veh_width) / 2.0);   // d = (veh_length - veh_width) / 2
  kp.veh_2r = (float)(2.0 * (0.5 * (double)d->veh_width));                       // 2 * r, r = 0.5 * veh_width
  {
    // veh3dof_tracking_detour_model.py:133-163 (1) / veh3dof_tracking_surrcstr_model.py:88,138-171 (2)
    const float det[7] = {10.f, 10.f, 500.f, 5.f, 1000.f, 1000.f, 50.f}, sur[7] = {0.04f, 0.04f, 0.02f, 0.02f, 0.01f, 0.01f, 0.01f};
    const bool sc = d->veh_detour == 2;
    for (int i = 0; i < 7; ++i) kp.veh_rc[i] = sc ? sur[i] : det[i];
    kp.veh_rscale = sc ? 1.f : 0.01f;
    kp.veh_roff = sc ? 0.f : 2.f;
    kp.veh_ydone = sc ? 2.f : 3.f;
    if (sc) kp.veh_2r = (float)(2.0 * (sqrt(2.0) / 2.0 * (double)d->veh_width));   // r = np.sqrt(2) / 2 * veh_width
  }
  kp.veh_Pdt = (float)((double)d->veh_pre_horizon * 0.1);   // self.pre_horizon * self.dt

  cudaError_t e = cudaGetDevice(&pl->device);
  cudaDeviceProp prop;
  if (e == cudaSuccess) e = cudaGetDeviceProperties(&prop, pl->device);
  if (e != cudaSuccess) { delete pl; return fail(std::string("no CUDA device: ") + cudaGetErrorString(e)); }
  if (prop.major != 9 || prop.minor != 0) { delete pl; return fail("gops_b200 is built for sm_90a and needs an H100-class (sm_90) device"); }
  pl->sm_count = prop.multiProcessorCount;
  pl->max_smem = (int)prop.sharedMemPerBlockOptin;

  std::vector<float> gp(d->horizon + 1);
  for (int k = 0; k <= d->horizon; ++k) gp[k] = (float)pow((double)d->gamma, (double)k);
  // note: python evaluates `gamma ** k` on the python float the caller passed; d->gamma is that value
  // rounded to fp32, so callers that need bit parity for non-representable gammas can update gpow via
  // gops_b200_plan_set_gamma (below) with the double value.
  if (cudaMalloc(&pl->gpow, gp.size() * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&pl->blob_pol, kp.w_floats * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&pl->blob_val, kp.w_floats * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&pl->blob_vtg, kp.w_floats * sizeof(float)) != cudaSuccess) {
    gops_b200_plan_destroy(pl);
    return fail("cudaMalloc failed for plan scratch");
  }
  if (cudaMemcpy(pl->gpow, gp.data(), gp.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
    gops_b200_plan_destroy(pl);
    return fail("cudaMemcpy(gpow) failed");
  }
  if (kp.obs_scaling) {
    const int od = d->policy.in_dim;
    if (cudaMalloc(&pl->osc, 2 * od * sizeof(float)) != cudaSuccess) { gops_b200_plan_destroy(pl); return fail("cudaMalloc failed"); }
    if (cudaMemcpy(pl->osc, d->obs_scale, od * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(pl->osc + od, d->obs_shift, od * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
      gops_b200_plan_destroy(pl);
      return fail("cudaMemcpy(obs scale/shift) failed");
    }
    kp.osc = pl->osc;
    kp.osh = pl->osc + od;
  }
  // wgmma rollout kernel: 64-wide nets whose inputs fit one 16-wide K block, state == obs models
  if (kp.hid == 64 && kp.pol.in <= tcf::K1 && (!infadp || kp.val.in <= tcf::K1) && rollout_fn_tc2(d->model, d->alg)) {
    make_net_tcf(kp.pol, pl->pol_tcf);
    if (infadp) make_net_tcf(kp.val, pl->val_tcf); else pl->val_tcf = pl->pol_tcf;
    pl->w_floats_tcf = pl->pol_tcf.blob > pl->val_tcf.blob ? pl->pol_tcf.blob : pl->val_tcf.blob;
    const size_t nb = (size_t)pl->w_floats_tcf * sizeof(float);
    if (cudaMalloc(&pl->blob_pol_tcf, nb) != cudaSuccess || cudaMalloc(&pl->blob_val_tcf, nb) != cudaSuccess ||
        cudaMalloc(&pl->blob_vtg_tcf, nb) != cudaSuccess) {
      gops_b200_plan_destroy(pl);
      return fail("cudaMalloc failed for plan scratch (wgmma rollout blobs)");
    }
    cudaMemset(pl->blob_pol_tcf, 0, nb); cudaMemset(pl->blob_val_tcf, 0, nb); cudaMemset(pl->blob_vtg_tcf, 0, nb);
    pl->tc_ok = true;
  }
  cudaMemset(pl->blob_pol, 0, kp.w_floats * sizeof(float));
  cudaMemset(pl->blob_val, 0, kp.w_floats * sizeof(float));
  cudaMemset(pl->blob_vtg, 0, kp.w_floats * sizeof(float));
  kp.gpow = pl->gpow;
  kp.blob_pol = pl->blob_pol; kp.blob_val = pl->blob_val; kp.blob_vtg = pl->blob_vtg;
  *out = pl;
  return 0;
}

int gops_b200_plan_set_gamma(gops_b200_plan* pl, double gamma) {
  if (!pl) return fail("null plan");
  DevGuard dg(pl->device);
  std::vector<float> gp(pl->kp.horizon + 1);
  for (int k = 0; k <= pl->kp.horizon; ++k) gp[k] = (float)pow(gamma, (double)k);
  pl->kp.gamma = (float)gamma;
  CUDA_OK(cudaMemcpy(pl->gpow, gp.data(), gp.size() * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

int gops_b200_plan_enable_timing(gops_b200_plan* pl, int enable) {
  if (!pl) return fail("null plan");
  DevGuard dg(pl->device);
  if (enable && !pl->ev0) {
    CUDA_OK(cudaEventCreate(&pl->ev0));
    CUDA_OK(cudaEventCreate(&pl->ev1));
  }
  pl->timing = enable != 0;
  return 0;
}

int gops_b200_plan_last_kernel_ms(gops_b200_plan* pl, float* ms) {
  if (!pl || !ms || !pl->ev0) return fail("timing not enabled");
  CUDA_OK(cudaEventSynchronize(pl->ev1));
  CUDA_OK(cudaEventElapsedTime(ms, pl->ev0, pl->ev1));
  return 0;
}

int gops_b200_plan_set_path(gops_b200_plan* pl, int path) {
  if (!pl) return fail("null plan");
  if (path != GOPS_PATH_AUTO && path != GOPS_PATH_MMA && path != GOPS_PATH_TC) return fail("unknown kernel path");
  if (path == GOPS_PATH_TC && !pl->tc_ok && !(pl->kp.hid > 64 && pl->desc.alg == GOPS_ALG_FHADP && lw_fn(pl->desc.model, 0)))
    return fail("the wgmma rollout kernel is not built for this plan (needs 64-wide nets, <= 16 inputs, idpendulum / lq)");
  pl->path = path;
  return 0;
}
int gops_b200_plan_last_path(const gops_b200_plan* pl) { return pl ? pl->last_path : -1; }

int gops_b200_plan_set_constraint(gops_b200_plan* pl, int mode, float coef) {
  if (!pl) return fail("null plan");
  if (mode < 0 || mode > 3) return fail("unknown constraint mode");
  const bool provider = (pl->desc.model == GOPS_MODEL_VEH3DOFCONTI && pl->desc.veh_errcstr) ||
                        (pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING && pl->desc.veh_detour);
  if (mode != 0 && !(provider && pl->desc.alg == GOPS_ALG_FHADP))
    return fail("constrained FHADP variants are built for the info['constraint'] providers pyth_veh3dofconti_errcstr and "
                "veh3dof_tracking_detour only");
  if (mode != 0 && !(coef > 0.f)) return fail("constraint coefficient must be positive");
  pl->kp.cstr_mode = mode;
  pl->kp.cstr_coef = coef;
  return 0;
}

int gops_b200_plan_launch_info(const gops_b200_plan* pl, int32_t* out4) {
  if (!pl || !out4) return fail("null argument");
  out4[0] = pl->last_grid; out4[1] = pl->last_NT; out4[2] = pl->last_S; out4[3] = (int32_t)pl->last_smem;
  return 0;
}

int gops_b200_plan_destroy(gops_b200_plan* pl) {
  ENTRY("gops_b200_plan_destroy(gops_b200_plan* p");
  if (!pl) return 0;
  DevGuard dg(pl->device);
  if (pl->ev0) { cudaEventDestroy(pl->ev0); cudaEventDestroy(pl->ev1); }
  if (pl->lw_exec) cudaGraphExecDestroy(pl->lw_exec);
  if (pl->lw_cap_stream) cudaStreamDestroy(pl->lw_cap_stream);
  if (pl->lw_net) gops_b200_mlpnet_destroy(pl->lw_net);
  {
    float* lw[] = {pl->lw_S, pl->lw_Dn, pl->lw_X, pl->lw_Z, pl->lw_Zb, pl->lw_lam, pl->lw_vacc, pl->lw_dX, pl->lw_sp, pl->lw_cacc,
                   pl->lw_xcar};
    for (float* q : lw) cudaFree(q);
    (void)cudaGetLastError();
  }
  void* ptrs[] = {pl->gpow, pl->blob_pol, pl->blob_val, pl->blob_vtg, pl->tape, pl->partial, pl->ext_ref, pl->xbuf, pl->osc,
                  pl->blob_tc, pl->blob_pol_tcf, pl->blob_val_tcf, pl->blob_vtg_tcf};
  const char* names[] = {"gpow", "blob_pol", "blob_val", "blob_vtg", "tape", "partial", "ext_ref", "xbuf", "osc", "blob_tc",
                         "blob_pol_tcf", "blob_val_tcf", "blob_vtg_tcf"};
  if (getenv("GOPS_B200_DEBUG")) {
    fprintf(stderr, "[gops_b200] destroy plan %p alg %d model %d:", (void*)pl, pl->desc.alg, pl->desc.model);
    for (size_t i = 0; i < sizeof(ptrs) / sizeof(ptrs[0]); ++i) fprintf(stderr, " %s=%p", names[i], ptrs[i]);
    fprintf(stderr, "\n");
  }
  static_assert(sizeof(ptrs) / sizeof(ptrs[0]) == sizeof(names) / sizeof(names[0]), "one name per buffer");
  for (size_t i = 0; i < sizeof(ptrs) / sizeof(ptrs[0]); ++i) {
    const cudaError_t e = cudaFree(ptrs[i]);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      if (getenv("GOPS_B200_DEBUG")) fprintf(stderr, "[gops_b200] cudaFree(%s) failed: %s\n", names[i], cudaGetErrorString(e));
    }
  }
  delete pl;
  return 0;
}

int64_t gops_b200_plan_param_count(const gops_b200_plan* pl, int which) {
  if (!pl) return -1;
  return which == 0 ? pl->kp.pol.nparam : pl->kp.val.nparam;
}

int gops_b200_rollout_grad(gops_b200_plan* pl, const gops_b200_batch* b, const float* policy_params,
                           const float* value_params, const float* vtarget_params, float inv_batch_global,
                           float* grad_out, float* scalars_out, void* stream) {
  ENTRY("float* grad_out, float* scalars_out, voi");
  if (!pl || !policy_params || !grad_out || !scalars_out) return fail("null argument");
  DevGuard dg(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int alg = pl->desc.alg;
  if (b && b->batch > 0 && b->obs && b->done && rollout_use_layerwise(pl, alg)) {
    if (pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING) {
      if (!b->state || !b->reference) return fail("veh3dof_tracking needs state (robot_state) and reference");
      if (b->ref_t < 0 || b->ref_t + pl->kp.horizon + pl->kp.veh_P + 1 > b->ref_len)
        return fail("veh3dof_tracking: reference too short for t + horizon + pre_horizon + 1 points");
      if (pl->desc.veh_detour && (!b->surr || b->ref_t + pl->kp.horizon + 1 > b->surr_len))
        return fail("veh3dof_tracking_detour needs the surrounding-vehicle predictions (ContextState.constraint), t + horizon + 1 points");
    }
    pl->kp.inv_B = inv_batch_global;
    return launch_rollout_layerwise(pl, b, policy_params, st, grad_out, scalars_out);
  }
  const bool tcr = b && rollout_use_tc(pl, b->batch);
  if (tcr ? launch_pack_tcf(policy_params, pl->pol_tcf, pl->blob_pol_tcf, st)
          : launch_pack(policy_params, pl->kp.pol, pl->kp.hid, pl->blob_pol, st)) return 1;
  if (alg != GOPS_ALG_FHADP) {
    if (!vtarget_params) return fail("vtarget_params required for INFADP");
    if (tcr ? launch_pack_tcf(vtarget_params, pl->val_tcf, pl->blob_vtg_tcf, st)
            : launch_pack(vtarget_params, pl->kp.val, pl->kp.hid, pl->blob_vtg, st)) return 1;
  }
  if (alg == GOPS_ALG_INFADP_VALUE) {
    if (!value_params) return fail("value_params required for INFADP value update");
    if (tcr ? launch_pack_tcf(value_params, pl->val_tcf, pl->blob_val_tcf, st)
            : launch_pack(value_params, pl->kp.val, pl->kp.hid, pl->blob_val, st)) return 1;
  }
  pl->kp.inv_B = inv_batch_global;
  pl->kp.tr_obs = pl->kp.tr_act = pl->kp.tr_rew = pl->kp.tr_done = nullptr;
  return launch_rollout(pl, b, alg, st, grad_out, scalars_out);
}

int gops_b200_rollout_trace(gops_b200_plan* pl, const gops_b200_batch* b, const float* policy_params, float* obs_out,
                            float* act_out, float* rew_out, float* done_out, void* stream) {
  ENTRY("float* act_out, float* rew_out, float* d");
  if (!pl || !policy_params) return fail("null argument");
  DevGuard dg(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  const bool tcr = b && rollout_use_tc(pl, b->batch);
  if (tcr ? launch_pack_tcf(policy_params, pl->pol_tcf, pl->blob_pol_tcf, st)
          : launch_pack(policy_params, pl->kp.pol, pl->kp.hid, pl->blob_pol, st)) return 1;
  pl->kp.inv_B = 1.f;
  pl->kp.tr_obs = obs_out; pl->kp.tr_act = act_out; pl->kp.tr_rew = rew_out; pl->kp.tr_done = done_out;
  return launch_rollout(pl, b, ALG_TRACE, st, nullptr, nullptr);
}

// wgmma inference (mlp_tc.cuh).  GOPS_B200_INFER=tc|mma forces one of the two 64-wide paths.
static bool infer_use_tc(const gops_b200_plan* pl, int64_t batch, int use_val) {
  if (pl->kp.hid != 64) return false;
  const char* e = getenv("GOPS_B200_INFER");
  if (e && !strcmp(e, "mma")) return false;
  // the wgmma inference kernel keeps the input planes in shared memory: wide inputs stay on the mma.sync kernel
  // whatever the batch size is (no batch-dependent failure)
  const NetL& L = use_val ? pl->kp.val : pl->kp.pol;
  TcNet T;
  memset(&T, 0, sizeof(T));
  T.k1 = L.in8;
  T.blob = 2 * 64 * T.k1 + 2 * 64 * 64 + round4(L.out * 64) + 64 + 64 + 4;
  if (tc_infer_smem_bytes(T, 1) > (size_t)pl->max_smem) return false;
  if (e && !strcmp(e, "tc")) return true;
  return batch >= 4096;
}

static int infer_tc(gops_b200_plan* pl, const float* params, const NetL& L, const float* obs, int64_t batch,
                    float virtual_t, float* out, cudaStream_t st, bool squash) {
  TcNet T;
  memset(&T, 0, sizeof(T));
  T.in = L.in; T.obs = L.obs; T.out = L.out; T.hact = L.hact; T.time_input = L.time_input; T.k1 = L.in8;
  T.g_w1 = L.g_w1; T.g_b1 = L.g_b1; T.g_w2 = L.g_w2; T.g_b2 = L.g_b2; T.g_w3 = L.g_w3; T.g_b3 = L.g_b3;
  int o = 0;
  T.o_w1h = o; o += 64 * T.k1;
  T.o_w1l = o; o += 64 * T.k1;
  T.o_w2h = o; o += 64 * 64;
  T.o_w2l = o; o += 64 * 64;
  T.o_w3 = o; o += round4(T.out * 64);
  T.o_b1 = o; o += 64;
  T.o_b2 = o; o += 64;
  T.o_b3 = o; o += 4;
  T.blob = o;
  T.squash = squash ? 1 : 0;
  for (int j = 0; j < MAXA; ++j) { T.half[j] = pl->kp.pol_half[j]; T.mid[j] = pl->kp.pol_mid[j]; }
  const int wgs = tc_infer_smem_bytes(T, 2) <= (size_t)pl->max_smem ? 2 : 1;
  const size_t smem = tc_infer_smem_bytes(T, wgs);
  if (smem > (size_t)pl->max_smem) return fail("wgmma inference: input width does not fit in shared memory");
  if (pl->blob_tc_floats < T.blob) {
    if (pl->blob_tc) cudaFree(pl->blob_tc);
    pl->blob_tc = nullptr; pl->blob_tc_floats = 0;
    CUDA_OK(cudaMalloc(&pl->blob_tc, (size_t)T.blob * sizeof(float)));
    pl->blob_tc_floats = T.blob;
  }
  pack_params_tc_kernel<<<8, 256, 0, st>>>(params, T, pl->blob_tc);
  ++g_launches;
  CUDA_OK_L(cudaGetLastError(), "launch#tc-pack");
  static bool attr_of[kMaxDevices] = {};     // function attributes are per device
  bool& attr = attr_of[pl->device >= 0 && pl->device < kMaxDevices ? pl->device : 0];
  if (!attr) {
    CUDA_OK(cudaFuncSetAttribute(mlp_infer_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, pl->max_smem));
    CUDA_OK(cudaFuncSetAttribute(mlp_infer_tc_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, pl->max_smem));
    attr = true;
  }
  const long long tiles = (batch + TC_TILE - 1) / TC_TILE;
  const long long ctas = (tiles + wgs - 1) / wgs;
  const int grid = (int)(ctas < pl->sm_count ? ctas : pl->sm_count);
  if (wgs == 2) mlp_infer_tc_kernel<2><<<grid, 256, smem, st>>>(T, pl->blob_tc, obs, batch, virtual_t, out);
  else mlp_infer_tc_kernel<1><<<grid, 128, smem, st>>>(T, pl->blob_tc, obs, batch, virtual_t, out);
  ++g_launches;
  CUDA_OK_L(cudaGetLastError(), "launch#tc-infer");
  return 0;
}

static int infer_common(gops_b200_plan* pl, const float* params, int use_val, const float* obs, int64_t batch,
                        float virtual_t, float* out, void* stream, bool squash) {
  if (!pl || !params || !obs || !out) return fail("null argument");
  if (batch <= 0) return fail("empty batch");
  DevGuard dg(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  const NetL& L = use_val ? pl->kp.val : pl->kp.pol;
  if (infer_use_tc(pl, batch, use_val)) return infer_tc(pl, params, L, obs, batch, virtual_t, out, st, squash);
  float* blob = use_val ? pl->blob_val : pl->blob_pol;
  if (launch_pack(params, L, pl->kp.hid, blob, st)) return 1;
  const int cfg = pick_config(pl, batch, true);
  if (cfg < 0) return fail("no kernel configuration fits in shared memory");
  const int S = config_of(pl, cfg).S, NTc = config_of(pl, cfg).NT;
  const long long tiles = (batch + NTc - 1) / NTc;
  const int grid = (int)(tiles < pl->sm_count ? tiles : pl->sm_count);
  const size_t smem = infer_smem_bytes(pl->kp, S, NTc);
  (void)S;
#define LAUNCH_INFER(HH, SS, NN)                                                                                  \
  do {                                                                                                        \
    CUDA_OK(cudaFuncSetAttribute(mlp_infer_kernel<HH, SS, NN>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                 pl->max_smem));                                                              \
    mlp_infer_kernel<HH, SS, NN><<<grid, NN, smem, st>>>(pl->kp, blob, use_val, obs, batch, virtual_t,        \
                                                         squash ? 1 : 0, out);                               \
    ++g_launches;                                                                                             \
  } while (0)
  if (pl->kp.hid > 64) {
    if ((size_t)grid * pl->kp.inp_max * (NTc + 4) > pl->xbuf_floats) {
      if (pl->xbuf) cudaFree(pl->xbuf);
      pl->xbuf = nullptr; pl->xbuf_floats = 0;
      const size_t need = (size_t)pl->sm_count * pl->kp.inp_max * (NTc + 4);
      CUDA_OK(cudaMalloc(&pl->xbuf, need * sizeof(float)));
      CUDA_OK(cudaMemset(pl->xbuf, 0, need * sizeof(float)));
      pl->xbuf_floats = need;
    }
    pl->kp.xbuf = pl->xbuf;
    LAUNCH_INFER(256, 32, 256);
  } else if (cfg == 0) LAUNCH_INFER(64, 128, 512);
  else if (cfg == 1) LAUNCH_INFER(64, 64, 256);
  else LAUNCH_INFER(64, 32, 128);
#undef LAUNCH_INFER
  CUDA_OK_L(cudaGetLastError(), "launch#4");
  return 0;
}

int gops_b200_policy_forward(gops_b200_plan* pl, const float* policy_params, const float* obs, int64_t batch,
                             float virtual_t, float* act_out, void* stream) {
  return infer_common(pl, policy_params, 0, obs, batch, virtual_t, act_out, stream, true);
}

int gops_b200_value_forward(gops_b200_plan* pl, const float* value_params, const float* obs, int64_t batch,
                            float* v_out, void* stream) {
  if (pl && pl->desc.alg == GOPS_ALG_FHADP) return fail("plan has no value network");
  return infer_common(pl, value_params, 1, obs, batch, 0.f, v_out, stream, false);
}

int gops_b200_mlp_forward(const gops_b200_mlp_desc* net, const float* params, const float* obs, int64_t batch,
                          float virtual_t, const float* act_low, const float* act_high, float* out, void* stream) {
  ENTRY("float virtual_t, const float* act_low, c");
  if (!net || !params || !obs || !out) return fail("null argument");
  if (batch <= 0) return fail("empty batch");
  const int dev = device_of(params);
  if (dev < 0 || dev >= kMaxDevices) return fail("device index out of range");
  DevGuard dg(dev);
  static thread_local gops_b200_plan* scratch_of[kMaxDevices] = {};   // reusable staging blob per host thread and device
  static thread_local int scratch_floats_of[kMaxDevices] = {};
  gops_b200_plan*& scratch = scratch_of[dev];
  int& scratch_floats = scratch_floats_of[dev];
  gops_b200_plan tmp;
  tmp.device = dev;
  KParams& kp = tmp.kp;
  memset(&kp, 0, sizeof(kp));
  std::string why;
  if (!make_net(*net, kp.pol, why)) return fail(why);
  kp.val = kp.pol;
  kp.hid = net->hidden;
  kp.w_floats = kp.pol.blob;
  kp.inp_max = kp.pol.inp;
  for (int j = 0; j < net->out_dim; ++j) {
    kp.pol_half[j] = act_low ? (act_high[j] - act_low[j]) / 2.f : 1.f;
    kp.pol_mid[j] = act_low ? (act_high[j] + act_low[j]) / 2.f : 0.f;
  }
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, dev));
  tmp.sm_count = prop.multiProcessorCount;
  tmp.max_smem = (int)prop.sharedMemPerBlockOptin;
  if (!scratch || scratch_floats < kp.w_floats) {
    if (scratch) { cudaFree(scratch->blob_pol); delete scratch; }
    scratch = new gops_b200_plan();
    scratch_floats = kp.w_floats;
    CUDA_OK(cudaMalloc(&scratch->blob_pol, (size_t)scratch_floats * sizeof(float)));
  }
  tmp.blob_pol = scratch->blob_pol;
  tmp.xbuf = scratch->xbuf;
  tmp.xbuf_floats = scratch->xbuf_floats;
  tmp.blob_tc = scratch->blob_tc;
  tmp.blob_tc_floats = scratch->blob_tc_floats;
  const int rc = infer_common(&tmp, params, 0, obs, batch, virtual_t, out, stream, act_low != nullptr);
  scratch->xbuf = tmp.xbuf;              // infer_common may have (re)allocated the wide-net scratch
  scratch->xbuf_floats = tmp.xbuf_floats;
  scratch->blob_tc = tmp.blob_tc;
  scratch->blob_tc_floats = tmp.blob_tc_floats;
  tmp.blob_pol = nullptr;
  tmp.xbuf = nullptr;
  tmp.blob_tc = nullptr;
  return rc;
}

int gops_b200_model_step(gops_b200_plan* pl, const gops_b200_batch* b, const float* action, float* next_obs,
                         float* reward, float* next_done, float* next_state, float* next_ref_points,
                         float* next_ref_time, void* stream) {
  ENTRY("float* next_ref_time, void* stream) {");
  if (!pl || !b || !action || !next_obs || !reward || !next_done) return fail("null argument");
  if (b->batch <= 0 || !b->obs || !b->done) return fail("bad batch");
  DevGuard dg(pl->device);
  KParams& kp = pl->kp;
  kp.batch = b->batch; kp.obs = b->obs; kp.done = b->done;
  const unsigned grid = (unsigned)((b->batch + 127) / 128);
  cudaStream_t st = (cudaStream_t)stream;
  const int act_dim = pl->desc.policy.out_dim;
  if (pl->desc.model == GOPS_MODEL_VEH3DOFCONTI || pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING) {
    const bool conti = pl->desc.model == GOPS_MODEL_VEH3DOFCONTI;
    if (!b->state || !next_state) return fail("model_step: vehicle models need state and next_state");
    if (conti && (!b->ref_points || !b->path_num || !b->u_num || !b->ref_time || !next_ref_points || !next_ref_time))
      return fail("model_step: pyth_veh3dofconti needs ref_points, path_num, u_num, ref_time and their outputs");
    if (!conti && (!b->reference || b->ref_t < 0 || b->ref_t + kp.veh_P + 2 > b->ref_len))
      return fail("model_step: veh3dof_tracking reference too short for t + 1 + pre_horizon + 1 points");
    if (pl->desc.veh_detour && (!b->surr || b->ref_t + 2 > b->surr_len))
      return fail("model_step: veh3dof_tracking_detour needs the surrounding-vehicle predictions for t and t + 1");
    kp.state = b->state; kp.ref_points = b->ref_points; kp.path_num = b->path_num; kp.u_num = b->u_num;
    kp.ref_time = b->ref_time; kp.reference = b->reference; kp.ref_t = b->ref_t; kp.ref_len = b->ref_len;
    kp.surr = b->surr; kp.surr_len = b->surr_len;
    if (pl->desc.veh_detour) launch_veh_step_detour(kp, action, next_obs, reward, next_done, next_state, st);
    else if (conti) veh_step_kernel<1><<<grid, 128, 0, st>>>(kp, action, next_obs, reward, next_done, next_state,
                                                        next_ref_points, next_ref_time);
    else veh_step_kernel<2><<<grid, 128, 0, st>>>(kp, action, next_obs, reward, next_done, next_state,
                                                  next_ref_points, next_ref_time);
    ++g_launches;
    CUDA_OK_L(cudaGetLastError(), "veh_step launch");
    return 0;
  }
  StepFn fn = step_fn(pl->desc.model);
  if (!fn) return fail("model_step: env model kind not built into this library");
  fn<<<grid, 128, 0, st>>>(kp, action, act_dim, next_obs, reward, next_done);
  ++g_launches;
  CUDA_OK_L(cudaGetLastError(), "launch#5");
  return 0;
}

int gops_b200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                        int32_t step, double lr, double beta1, double beta2, double eps, void* stream) {
  ENTRY("int32_t step, double lr, double beta1, d");
  if (!params || !grads || !exp_avg || !exp_avg_sq) return fail("null argument");
  if (n <= 0 || step < 1) return fail("bad n/step");
  DevGuard dg(device_of(params));
  // python-side scalars of torch/optim/adam.py are doubles; only the tensor math is fp32
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  const float step_size = (float)(lr / bc1);
  const float bc2_sqrt = (float)sqrt(bc2);
  adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      params, grads, exp_avg, exp_avg_sq, n, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps,
      step_size, bc2_sqrt);
  ++g_launches;
  CUDA_OK_L(cudaGetLastError(), "launch#6");
  return 0;
}

int gops_b200_polyak(float* target, const float* src, float tau, int64_t n, void* stream) {
  ENTRY("int gops_b200_polyak(float* target, cons");
  if (!target || !src || n <= 0) return fail("bad argument");
  DevGuard dg(device_of(target));
  polyak_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(target, src, tau, n);
  ++g_launches;
  CUDA_OK_L(cudaGetLastError(), "launch#7");
  return 0;
}

}  // extern "C"
