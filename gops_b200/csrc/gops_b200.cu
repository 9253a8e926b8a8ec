// libgops_b200.so: C ABI (include/gops_b200.h) over the fused sm_90a rollout kernels.
#include "gops_b200.h"

#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <memory>
#include <new>
#include <string>
#include <vector>

#include "host_util.h"
#include "kernel.cuh"
#include "aux_kernels.cuh"
#include "mlp_tc.cuh"
#include "rollout_tc2.cuh"
#include "lw_rollout.cuh"
#include "model_kernels.cuh"
#include <cuda_bf16.h>

using namespace gops;

namespace {

int round4(int x) { return (x + 3) & ~3; }

// status of the launches just enqueued: "<label> cudaGetLastError(): <CUDA error>"
int launched(const char* label) {
  CUDA_OK(cudaGetLastError(), std::string(label) + " cudaGetLastError()");
  return 0;
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

Config config_of(int hid, int cfg) { return hid > 64 ? kWideConfig : kConfigs[cfg]; }

const ModelKernels* kernels_of(int model) {
  switch (model) {
    case GOPS_MODEL_IDPENDULUM: return &kernels_idp();
    case GOPS_MODEL_LQ: return &kernels_lq();
    case GOPS_MODEL_VEH3DOFCONTI: return &kernels_vehconti();
    case GOPS_MODEL_VEH3DOF_TRACKING: return &kernels_vehtrack();
    case GOPS_MODEL_MOBILEROBOT: return &kernels_mobilerobot();
    default: return nullptr;
  }
}
int model_ns(int model) {
  switch (model) {
    case GOPS_MODEL_LQ: return LQN;
    case GOPS_MODEL_VEH3DOFCONTI: return ModelVehConti::NS;
    case GOPS_MODEL_MOBILEROBOT: return ModelMobileRobot::NS;
    default: return 6;
  }
}

}  // namespace

struct gops_b200_plan {
  gops_b200_plan_desc desc;
  KParams kp;             // the plan's constants; every launch binds its batch and scratch into its own copy
  int device = 0, sm_count = 0, max_smem = 0;
  DevBuf gpow, blob_pol, blob_val, blob_vtg;
  DevBuf osc;             // obs scale | shift, 2 * obs_dim floats
  DevBuf tape, partial, ext_ref, xbuf;   // fused-kernel scratch
  DevBuf blob_tc;         // wgmma inference path: chunk-major hi / lo weight planes
  // wgmma rollout kernel (BF16x3): NetL with the bf16-plane blob offsets, packed blobs
  bool tc_ok = false;
  NetL pol_tcf, val_tcf;
  int w_floats_tcf = 0;
  DevBuf blob_pol_tcf, blob_val_tcf, blob_vtg_tcf;
  bool timing = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int path = GOPS_PATH_AUTO, last_path = 0;
  // layer-wise wgmma path of the wide nets (lw_rollout.cuh + dense_tc.cu)
  gops_b200_mlpnet* lw_net = nullptr;
  long long lw_cap = 0;
  DevBuf lw_S, lw_Dn, lw_X, lw_Z, lw_Zb, lw_lam, lw_vacc, lw_dX, lw_sp, lw_cacc, lw_xcar;
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

enum class Route { Layerwise, Tc, Mma };

// the layer-wise path is built for the plan: wide nets, FHADP, a model with layer-wise kernels
bool layerwise_built(const gops_b200_plan* pl) {
  return pl->kp.hid > 64 && pl->desc.alg == GOPS_ALG_FHADP && kernels_of(pl->desc.model)->lw.init;
}

// Kernel path of a rollout.  The plan option (gops_b200_plan_set_path) is overridden by GOPS_B200_ROLLOUT=tc|mma.
//  * layer-wise: FHADP with wide nets (AUTO or TC, horizon <= 128), and always FHADP2 (open loop) and the detour models;
//  * wgmma: wherever it is built for the plan (64-wide nets, <= 16 inputs, state == obs models), on TC or from 2^14
//    samples on AUTO;
//  * mma.sync otherwise (and the A/B baseline on MMA).
// Trace (ALG_TRACE) never takes the layer-wise path.
Route rollout_route(const gops_b200_plan* pl, int alg, long long batch) {
  int path = pl->path;
  const char* e = getenv("GOPS_B200_ROLLOUT");
  if (e && !strcmp(e, "mma")) path = GOPS_PATH_MMA;
  if (e && !strcmp(e, "tc")) path = GOPS_PATH_TC;
  if (pl->desc.open_loop || pl->desc.veh_detour) {
    if (alg == ALG_FHADP) return Route::Layerwise;
  } else if (alg == ALG_FHADP && pl->kp.horizon <= 128 && layerwise_built(pl) && path != GOPS_PATH_MMA) {
    return Route::Layerwise;
  }
  if (!pl->tc_ok || path == GOPS_PATH_MMA) return Route::Mma;
  if (path == GOPS_PATH_TC) return Route::Tc;
  // below ~2^14 samples the mma.sync kernel with its 32-sample tiles spreads the batch over more SMs and finishes
  // first.  Measured on one H100 80GB HBM3 (700 W) with the previous wgmma kernel (128-sample sub-tiles, one group per
  // SM), ms per update mma / wgmma: FHADP idpendulum H = 30  2^13 0.74 / 0.78, 2^14 1.20 / 0.78, 2^18 11.8 / 10.4;
  // INFADP lq s4a2 PEV + PIM  2^12 0.66 / 0.69, 2^14 0.86 / 0.71.  The current kernel (64-sample sub-tiles, three per
  // SM) is faster at 2^18; its crossover has not been re-measured.
  return batch >= 16384 ? Route::Tc : Route::Mma;
}

// The inputs a rollout of this plan needs, checked before anything is enqueued.
int check_batch(const gops_b200_plan* pl, const gops_b200_batch* b, bool layerwise) {
  if (!b || b->batch <= 0) return fail("empty batch");
  if (!b->obs || !b->done) return fail("obs/done pointers are required");
  if (pl->desc.model == GOPS_MODEL_VEH3DOFCONTI &&
      (!b->state || !b->ref_points || !b->path_num || !b->u_num || !b->ref_time))
    return fail("pyth_veh3dofconti needs state, ref_points, path_num, u_num, ref_time");
  if (pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING) {
    if (!b->state || !b->reference) return fail("veh3dof_tracking needs state (robot_state) and reference");
    if (b->ref_t < 0 || b->ref_t + pl->kp.horizon + pl->kp.veh_P + 1 > b->ref_len)
      return fail("veh3dof_tracking: reference too short for t + horizon + pre_horizon + 1 points");
    if (layerwise && pl->desc.veh_detour && (!b->surr || b->ref_t + pl->kp.horizon + 1 > b->surr_len))
      return fail("veh3dof_tracking_detour needs the surrounding-vehicle predictions (ContextState.constraint), t + horizon + 1 points");
  }
  if (pl->desc.model == GOPS_MODEL_MOBILEROBOT && !pl->kp.noise)
    return fail("pyth_mobilerobot needs its obstacle noise [horizon][batch][2] (gops_b200_plan_set_model_io)");
  return 0;
}

// KParams of one launch: the plan's constants and this call's batch
KParams bind_batch(const gops_b200_plan* pl, const gops_b200_batch* b, int alg) {
  KParams p = pl->kp;
  p.alg = alg;
  p.batch = b->batch;
  p.obs = b->obs; p.done = b->done; p.state = b->state; p.ref_points = b->ref_points;
  p.path_num = b->path_num; p.u_num = b->u_num; p.ref_time = b->ref_time; p.reference = b->reference;
  p.ref_t = b->ref_t; p.ref_len = b->ref_len;
  p.surr = b->surr; p.surr_len = b->surr_len;
  return p;
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

// weights of one network into the blob layout of the rollout kernel taking `route`
int launch_pack(const gops_b200_plan* pl, Route route, const float* flat, bool value_net, float* blob, float* blob_tcf,
                cudaStream_t st) {
  if (route == Route::Tc) {
    pack_params_tcf_kernel<<<8, 256, 0, st>>>(flat, value_net ? pl->val_tcf : pl->pol_tcf, blob_tcf);
    ++g_launches;
    return launched("launch#tcf-pack");
  }
  pack_params_kernel<<<pl->kp.hid > 64 ? 64 : 8, 256, 0, st>>>(flat, value_net ? pl->kp.val : pl->kp.pol, pl->kp.hid, blob);
  ++g_launches;
  return launched("launch#1");
}

int pick_config(const KParams& kp, int sm_count, int max_smem, long long B, bool infer) {
  if (kp.hid > 64) return 0;
  // the largest chunk (threads per CTA) that still gives every SM at least one CTA
  const char* force = getenv("GOPS_B200_CFG");
  auto fits = [&](int c) {
    const size_t sm = infer ? infer_smem_bytes(kp, kConfigs[c].S, kConfigs[c].NT)
                            : rollout_smem_bytes(kp, kConfigs[c].S, kConfigs[c].NT);
    return sm <= (size_t)max_smem;
  };
  if (force && force[0] >= '0' && force[0] <= '2' && fits(force[0] - '0')) return force[0] - '0';
  int best = -1;
  for (int c = 0; c < 3; ++c) {
    if (!fits(c)) continue;
    best = c;
    if (B >= (long long)sm_count * kConfigs[c].NT) return c;
  }
  return best;
}

// grow-only scratch of the fused kernels: tape [grid][H][tape_ch][NT], vehicle reference windows, wide-net observation
// tiles and the gradient partials
int ensure_scratch(gops_b200_plan* pl, int grid, int NT, int H, int tape_ch, size_t partial_floats) {
  if (pl->tape.ensure((size_t)grid * H * tape_ch * NT)) return 1;
  if (pl->desc.model == GOPS_MODEL_VEH3DOFCONTI && pl->ext_ref.ensure((size_t)grid * (pl->kp.veh_P + 1 + H) * 4 * NT, true))
    return 1;
  if (pl->kp.hid > 64 && pl->xbuf.ensure((size_t)grid * pl->kp.inp_max * (NT + 4), true)) return 1;
  return pl->partial.ensure(partial_floats);
}

// One fused rollout kernel (wgmma or mma.sync) and, unless tracing, the reduction of its gradient partials.
int launch_fused(gops_b200_plan* pl, KParams p, Route route, cudaStream_t st, float* grad_out, float* scalars_out) {
  const bool tc = route == Route::Tc;
  const int alg = p.alg;
  const ModelKernels& K = *kernels_of(pl->desc.model);
  RolloutFn fn;
  int S, NT, tape_cols, rows;      // rows: gradient partial rows (= independent warpgroups) per CTA
  // wgmma: one CTA per SM (shared memory); a batch of fewer sub-tiles than SMs gets one CTA per sub-tile, so that it
  // spreads over the SMs (the kernel leaves the other warpgroups of such a CTA idle)
  long long slots = pl->sm_count;  // CTAs resident at once
  if (tc) {
    const int hact = (alg == ALG_FHADP || pl->pol_tcf.hact == pl->val_tcf.hact) ? pl->pol_tcf.hact : -1;
    // the fixed-chain kernel, where the model has one, is built for nets with one output (val_tcf = pol_tcf on FHADP)
    const bool chain = K.tc[kTcGeluChain][alg] && wrap_bits(p) == kTcChain && pl->pol_tcf.out == 1 && pl->val_tcf.out == 1;
    fn = K.tc[hact != GOPS_ACT_GELU ? kTcGeneric : chain ? kTcGeluChain : kTcGelu][alg];
    if (!fn) return fail("wgmma rollout kernel not built for this env model");
    p.pol = pl->pol_tcf;
    p.val = pl->val_tcf;
    p.blob_pol = pl->blob_pol_tcf.p; p.blob_val = pl->blob_val_tcf.p; p.blob_vtg = pl->blob_vtg_tcf.p;
    p.w_floats = pl->w_floats_tcf;
  }
  const NetL& upd = (alg == ALG_PEV) ? p.val : p.pol;
  p.part_stride = round4(upd.nparam + 4);
  p.dw_floats = round4(upd.nacc);
  // tape columns per step: state, done flag, then per policy output z (mma.sync) or the action a and d a / d z (wgmma)
  p.tape_ch = model_ns(pl->desc.model) + 1 + (tc ? 2 : 1) * p.pol.out;
  size_t smem;
  if (tc) {
    S = tc2::GT; NT = tc2::NT2; tape_cols = tc2::WGS * tc2::GT; rows = tc2::WGS;
    smem = tc2::smem_bytes(p.w_floats);
    if (smem > (size_t)pl->max_smem) return fail("wgmma rollout kernel does not fit in shared memory");
    if (allow_smem((const void*)fn, pl->device, pl->max_smem)) return 1;
  } else {
    const int cfg = pick_config(p, pl->sm_count, pl->max_smem, p.batch, false);
    if (cfg < 0) return fail("no kernel configuration fits in shared memory");
    S = config_of(p.hid, cfg).S; NT = tape_cols = config_of(p.hid, cfg).NT; rows = 1;
    fn = K.mma[p.hid > 64][cfg][alg];
    if (!fn) return fail("env model kind not built into this library");
    smem = rollout_smem_bytes(p, S, NT);
    if (smem > (size_t)pl->max_smem) return fail("rollout kernel does not fit in shared memory");
    if (allow_smem((const void*)fn, pl->device, pl->max_smem)) return 1;
    int occ = 1;
    CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, NT, smem));
    if (occ < 1) return fail("rollout kernel does not fit on an SM");
    // one CTA per SM slot as long as every CTA still gets at least one S-sample sub-tile: the kernel splits the
    // batch into balanced contiguous ranges, so small batches spread over all SMs with partially filled chunks
    slots *= occ;
  }
  p.n_tiles = (int)((p.batch + NT - 1) / NT);
  const long long subtiles = (p.batch + S - 1) / S;
  const int grid = (int)(subtiles < slots ? subtiles : slots);
  if (ensure_scratch(pl, grid, tape_cols, p.horizon, p.tape_ch, (size_t)grid * rows * p.part_stride)) return 1;
  p.tape = pl->tape.p;
  p.ext_ref = pl->ext_ref.p;
  p.xbuf = pl->xbuf.p;
  p.partial = pl->partial.p;
  if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev0, st));
  fn<<<grid, NT, smem, st>>>(p);
  ++g_launches;
  if (launched(tc ? "launch#2-tc" : "launch#2")) return 1;
  if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev1, st));
  pl->last_grid = grid; pl->last_S = S; pl->last_NT = NT; pl->last_smem = smem;
  pl->last_path = tc ? GOPS_PATH_TC : GOPS_PATH_MMA;
  if (alg != ALG_TRACE) {
    const int n = upd.nparam + 4;
    reduce_partials_kernel<<<(n + 255) / 256, 256, 0, st>>>(pl->partial.p, grid * rows, p.part_stride, upd.nparam, grad_out,
                                                           scalars_out);
    ++g_launches;
    if (launched(tc ? "launch#3-tc" : "launch#3")) return 1;
  }
  return 0;
}

// Buffers of the layer-wise path for batches up to B (capacity rounded up to 128 rows).  The policy mlpnet is
// recreated with them, and the captured graph (which holds the old buffers) dropped.
int ensure_lw(gops_b200_plan* pl, long long B, bool open) {
  if (pl->lw_net && B <= pl->lw_cap) return 0;
  const KParams& kp = pl->kp;
  const int H = kp.horizon, A = kp.pol.out, in = kp.pol.in, ldx = round4(in), NS = model_ns(pl->desc.model);
  if (pl->lw_net) gops_b200_mlpnet_destroy(pl->lw_net);
  pl->lw_net = nullptr;
  if (pl->lw_exec) { cudaGraphExecDestroy(pl->lw_exec); pl->lw_exec = nullptr; }
  pl->lw_key.clear();
  const size_t cap = (size_t)(B + 127) / 128 * 128;
  if (open) {       // FHADP2: one policy evaluation emits all H actions
    const int32_t sizes[4] = {in, pl->desc.policy.hidden, pl->desc.policy.hidden, A * H};
    if (gops_b200_mlpnet_create(sizes, 4, kp.pol.hact, cap, 1, &pl->lw_net)) return 1;
  } else {
    const int32_t sizes[4] = {in, kp.hid, kp.hid, A};
    if (gops_b200_mlpnet_create(sizes, 4, kp.pol.hact, cap, H, &pl->lw_net)) return 1;
    if (gops_b200_mlpnet_keep_deltas(pl->lw_net, 1)) return 1;
    if (pl->lw_X.ensure((H + 1) * cap * ldx) || pl->lw_dX.ensure(cap * ldx)) return 1;
    if (pl->desc.veh_detour && (pl->lw_cacc.ensure(3 * cap) || pl->lw_xcar.ensure(cap * ldx))) return 1;
  }
  if (pl->lw_S.ensure((H + 1) * NS * cap) || pl->lw_Dn.ensure((H + 1) * cap) || pl->lw_Z.ensure(H * cap * A) ||
      pl->lw_Zb.ensure(H * cap * A) || pl->lw_lam.ensure(NS * cap) || pl->lw_vacc.ensure(cap) || pl->lw_sp.ensure(2 * 256))
    return 1;
  pl->lw_cap = (long long)cap;
  return 0;
}

// Runs enqueue(stream) through the plan's CUDA graph: once the same call (same `key`) has been seen twice it is
// captured and replayed, which removes the launch gaps.  GOPS_B200_GRAPH=0 keeps every call eager.
template <class Enqueue>
int run_graphed(gops_b200_plan* pl, const std::vector<unsigned char>& key, cudaStream_t st, Enqueue&& enqueue) {
  if (pl->lw_exec && key == pl->lw_key) {
    CUDA_OK(cudaGraphLaunch(pl->lw_exec, st));
    g_launches += pl->lw_graph_launches;
    return 0;
  }
  if (key == pl->lw_key) ++pl->lw_key_hits;
  else {
    pl->lw_key = key;
    pl->lw_key_hits = 0;
    if (pl->lw_exec) { cudaGraphExecDestroy(pl->lw_exec); pl->lw_exec = nullptr; }
  }
  const char* ge = getenv("GOPS_B200_GRAPH");
  const bool graphs = !(ge && !strcmp(ge, "0"));
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
      return 0;
    }
    (void)cudaGetLastError();
    if (pl->lw_exec) { cudaGraphExecDestroy(pl->lw_exec); pl->lw_exec = nullptr; }
    pl->lw_graph_off = true;
    g_launches = n0;
  }
  return enqueue(st);
}

// Layer-wise FHADP update (wide nets, FHADP2, detour models): per-step rollout kernels around the wgmma policy MLP.
int launch_layerwise(gops_b200_plan* pl, const KParams& p, const float* policy_params, cudaStream_t st, float* grad_out,
                     float* scalars_out) {
  const int H = p.horizon, A = p.pol.out, ldx = round4(p.pol.in);
  const long long B = p.batch;
  const bool open = pl->desc.open_loop != 0, detour = pl->desc.veh_detour != 0;
  if (ensure_lw(pl, B, open)) return 1;
  const long long cap = pl->lw_cap;
  const LwKernels& lw = kernels_of(pl->desc.model)->lw;
  const LwFn f_init = lw.init, f_step = detour ? lw_fn_vehtrack_detour(1) : lw.step,
             f_rev = detour ? lw_fn_vehtrack_detour(2) : lw.reverse;
  LwArgs a;
  memset(&a, 0, sizeof(a));
  a.ldx = ldx; a.act_dim = A; a.bstride = cap;
  a.zs_k = open ? A : cap * A;          // Z / Zb: open loop [B][H A], closed loop [H][cap][A]
  a.zs_b = open ? (long long)H * A : A;
  a.S = pl->lw_S.p; a.Dn = pl->lw_Dn.p; a.X = open ? nullptr : pl->lw_X.p; a.Z = pl->lw_Z.p; a.Zb = pl->lw_Zb.p;
  a.lam = pl->lw_lam.p; a.vacc = pl->lw_vacc.p;
  if (!open) { a.cacc = pl->lw_cacc.p; a.xcar = pl->lw_xcar.p; }
  // S / Dn are indexed with the real batch as the row count
  const unsigned grid = (unsigned)((B + 127) / 128);
  const int sub = pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING ? LW_SUB : 1;
  const unsigned grid_step = (unsigned)((B * sub + 127) / 128);
  const int nb = 64;
  if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev0, st));
  if (open) {       // FHADP2: one policy evaluation emits all H actions; the rollout kernels read them strided
    if (gops_b200_mlpnet_pack(pl->lw_net, policy_params, st)) return 1;
    if (gops_b200_mlpnet_forward(pl->lw_net, p.obs, p.pol.obs, B, 0, 1, pl->lw_Z.p, H * A, st)) return 1;
    f_init<<<grid, 128, 0, st>>>(p, a);
    for (int k = 0; k < H; ++k) {
      a.k = k;
      f_step<<<grid_step, 128, 0, st>>>(p, a);
    }
    for (int k = H - 1; k >= 0; --k) {
      a.k = k;
      f_rev<<<grid, 128, 0, st>>>(p, a);
    }
    g_launches += 1 + 2 * H;
    if (gops_b200_mlpnet_backward(pl->lw_net, pl->lw_Zb.p, H * A, B, 0, grad_out, 0, nullptr, 0, st)) return 1;
    lw_scalars_kernel<<<nb, 256, 0, st>>>(pl->lw_vacc.p, pl->lw_Dn.p + (size_t)H * B, B, p.inv_B, pl->lw_sp.p);
    lw_scalars_final_kernel<<<1, 32, 0, st>>>(pl->lw_sp.p, nb, scalars_out);
    g_launches += 2;
    if (launched("open-loop rollout")) return 1;
  } else {
    // ~10 launches per horizon step, each a few microseconds: replayed as one CUDA graph (run_graphed)
    auto enqueue = [&](cudaStream_t st) -> int {
      if (gops_b200_mlpnet_pack(pl->lw_net, policy_params, st)) return 1;
      f_init<<<grid, 128, 0, st>>>(p, a);
      ++g_launches;
      if (detour) {
        CUDA_OK(cudaMemsetAsync(pl->lw_cacc.p, 0, sizeof(float) * 3 * (size_t)B, st));
        CUDA_OK(cudaMemsetAsync(pl->lw_xcar.p, 0, sizeof(float) * (size_t)B * ldx, st));
      }
      for (int k = 0; k < H; ++k) {
        if (gops_b200_mlpnet_forward(pl->lw_net, pl->lw_X.p + (size_t)k * cap * ldx, ldx, B, k, 1, pl->lw_Z.p + (size_t)k * cap * A,
                                     A, st))
          return 1;
        a.k = k;
        f_step<<<grid_step, 128, 0, st>>>(p, a);
        ++g_launches;
      }
      for (int k = H - 1; k >= 0; --k) {
        a.k = k;
        a.dX = k == H - 1 ? nullptr : pl->lw_dX.p;
        f_rev<<<grid, 128, 0, st>>>(p, a);
        ++g_launches;
        if (gops_b200_mlpnet_backward(pl->lw_net, pl->lw_Zb.p + (size_t)k * cap * A, A, B, k, nullptr, 0, k > 0 ? pl->lw_dX.p : nullptr,
                                      ldx, st))
          return 1;
      }
      if (gops_b200_mlpnet_wgrad_slots(pl->lw_net, 0, H, B, pl->lw_X.p, ldx, cap, pl->lw_Zb.p, A, cap, grad_out, 0, st)) return 1;
      if (detour) {
        lw_launch_scalars_detour(p, pl->lw_vacc.p, pl->lw_cacc.p, pl->lw_Dn.p + (size_t)H * B, scalars_out, st);
        g_launches += 1;
      } else {
        lw_scalars_kernel<<<nb, 256, 0, st>>>(pl->lw_vacc.p, pl->lw_Dn.p + (size_t)H * B, B, p.inv_B, pl->lw_sp.p);
        lw_scalars_final_kernel<<<1, 32, 0, st>>>(pl->lw_sp.p, nb, scalars_out);
        g_launches += 2;
      }
      return launched("layer-wise rollout");
    };
    std::vector<unsigned char> key(sizeof(KParams) + 4 * sizeof(void*));
    memcpy(key.data(), &p, sizeof(KParams));
    const void* kptr[4] = {policy_params, grad_out, scalars_out, (const void*)st};
    memcpy(key.data() + sizeof(KParams), kptr, sizeof(kptr));
    if (run_graphed(pl, key, st, enqueue)) return 1;
  }
  if (pl->timing) CUDA_OK(cudaEventRecord(pl->ev1, st));
  pl->last_grid = (int)grid; pl->last_S = 128; pl->last_NT = 128; pl->last_smem = 0; pl->last_path = GOPS_PATH_TC;
  return 0;
}

// The plan's constants from its descriptor; checks the descriptor in a fixed order and allocates nothing.
int plan_constants(const gops_b200_plan_desc* d, KParams& kp) {
  memset(&kp, 0, sizeof(kp));
  if (d->alg < GOPS_ALG_FHADP || d->alg > GOPS_ALG_INFADP_VALUE) return fail("unknown algorithm kind");
  if (d->horizon < 1 || d->horizon > 4096) return fail("horizon out of range");
  const ModelKernels* K = kernels_of(d->model);
  if (!K) return fail("env model kind not built into this library");
  std::string why;
  gops_b200_mlp_desc pol_desc = d->policy;
  if (d->open_loop) {
    if (d->alg != GOPS_ALG_FHADP) return fail("open_loop (FHADP2) needs alg = GOPS_ALG_FHADP");
    if (d->policy.time_input || d->policy.out_dim % d->horizon || d->policy.out_dim > 256)
      return fail("open_loop: policy.out_dim must be act_dim * horizon (<= 256), without time input");
    pol_desc.out_dim = d->policy.out_dim / d->horizon;      // kp.pol describes ONE step's action block
    if (pol_desc.hidden != 64 && pol_desc.hidden != 256) pol_desc.hidden = 256;   // geometry only; the mlpnet takes the real width
  }
  if (!make_net(pol_desc, kp.pol, why)) return fail("policy: " + why);
  const bool infadp = d->alg != GOPS_ALG_FHADP;
  if (infadp) {
    if (!make_net(d->value, kp.val, why)) return fail("value: " + why);
    if (d->value.out_dim != 1 || d->value.time_input) return fail("value net must be StateValue (out 1)");
    if (d->value.in_dim != d->policy.in_dim) return fail("value/policy obs dims differ");
  } else {
    kp.val = kp.pol;
  }
  const int act_dim = pol_desc.out_dim;
  int obs_dim_model = 0;
  if (d->model == GOPS_MODEL_IDPENDULUM) obs_dim_model = 6;
  if (d->model == GOPS_MODEL_LQ) {
    if (d->lq_n < 1 || d->lq_n > LQN || d->lq_m < 1 || d->lq_m > MAXA) return fail("lq dims out of range");
    obs_dim_model = d->lq_n;
    if (act_dim != d->lq_m) return fail("policy out_dim != lq action dim");
  }
  if (d->model == GOPS_MODEL_VEH3DOFCONTI || d->model == GOPS_MODEL_VEH3DOF_TRACKING) {
    // the vehicle models declare +-inf observation bounds (pyth_veh3dofconti_model.py:79-88): clip_obs is the identity
    if (d->veh_pre_horizon < 1) return fail("veh_pre_horizon must be >= 1");
    obs_dim_model = 6 + 4 * d->veh_pre_horizon + (d->veh_detour ? 4 : 0);
    if (act_dim != 2) return fail("vehicle models have 2 actions");
    if (d->veh_detour) {
      if (d->veh_detour != 1 && d->veh_detour != 2) return fail("veh_detour: 1 (detour) or 2 (surrcstr)");
      if (d->model != GOPS_MODEL_VEH3DOF_TRACKING || d->alg != GOPS_ALG_FHADP || d->open_loop)
        return fail("veh3dof_tracking_detour is built for FHADP and its constrained variants (closed-loop policy) only");
      if (d->obs_scaling) return fail("veh3dof_tracking_detour: ScaleObservation is not built");
      if (!(d->veh_length > d->veh_width) || !(d->veh_width > 0.f)) return fail("veh3dof_tracking_detour: need veh_length > veh_width > 0");
    }
  }
  if (d->model == GOPS_MODEL_MOBILEROBOT) {
    obs_dim_model = ModelMobileRobot::NS;
    if (act_dim != 2) return fail("pyth_mobilerobot has 2 actions");
    // the noise is drawn once per model step: a repeated step would need draws per repetition
    if (d->repeat_num > 1) return fail("repeat_num > 1 (ActionRepeat) is not built for pyth_mobilerobot");
  }
  if (d->policy.in_dim != obs_dim_model) return fail("policy in_dim does not match the env model obs_dim");
  if (d->model == GOPS_MODEL_IDPENDULUM && act_dim != 1) return fail("idpendulum has 1 action");

  kp.horizon = d->horizon;
  kp.hid = pol_desc.hidden;
  if (d->open_loop && !K->lw.init) return fail("open_loop (FHADP2) is not built for this env model");
  if (infadp && d->value.hidden != d->policy.hidden) return fail("policy and value hidden widths differ");
  kp.gamma = d->gamma;
  kp.w_floats = kp.pol.blob > kp.val.blob ? kp.pol.blob : kp.val.blob;
  kp.inp_max = kp.pol.inp > kp.val.inp ? kp.pol.inp : kp.val.inp;
  kp.dw_floats = round4(kp.pol.nacc > kp.val.nacc ? kp.pol.nacc : kp.val.nacc);
  kp.action_scale = d->action_scale; kp.clip_action = d->clip_action; kp.mask_at_done = d->mask_at_done;
  kp.reward_shaping = d->reward_shaping; kp.reward_shift = d->reward_shift; kp.reward_scale = d->reward_scale;
  kp.obs_scaling = d->obs_scaling ? 1 : 0;
  kp.repeat_num = (d->repeat_num > 0 && d->model != GOPS_MODEL_MOBILEROBOT) ? d->repeat_num : 0;
  kp.sum_reward = d->sum_reward ? 1 : 0;
  if (kp.repeat_num > 0 && !(d->model == GOPS_MODEL_IDPENDULUM || d->model == GOPS_MODEL_LQ))
    return fail("repeat_num (ActionRepeat) is supported for state==obs models only (not built for vehicle models)");
  if (kp.repeat_num > 16) return fail("repeat_num > 16 not supported");
  if (kp.obs_scaling && (!d->obs_scale || !d->obs_shift)) return fail("obs_scaling without obs_scale/obs_shift arrays");
  bool finite_obs_bound = false;
  for (int j = 0; j < MAXA; ++j) {
    kp.min_action[j] = d->min_action[j]; kp.max_action[j] = d->max_action[j];
    kp.act_low[j] = d->act_low[j]; kp.act_high[j] = d->act_high[j];
    // (act_high_lim - act_low_lim) / 2 and (act_high_lim + act_low_lim) / 2 in fp32, mlp.py:74-76
    kp.pol_half[j] = (d->pol_act_high[j] - d->pol_act_low[j]) / 2.f;
    kp.pol_mid[j] = (d->pol_act_high[j] + d->pol_act_low[j]) / 2.f;
  }
  const bool state_is_obs = d->model == GOPS_MODEL_IDPENDULUM || d->model == GOPS_MODEL_LQ;
  const bool robot = d->model == GOPS_MODEL_MOBILEROBOT;   // 13 bounds: the model's own (the descriptor carries 8)
  for (int f = 0; f < kMaxObs; ++f) {
    const bool in = f < obs_dim_model;
    kp.obs_low[f] = (robot && in) ? kRobotObsLow[f] : (state_is_obs && in && f < LQN) ? d->obs_low[f] : -INFINITY;
    kp.obs_high[f] = (robot && in) ? kRobotObsHigh[f] : (state_is_obs && in && f < LQN) ? d->obs_high[f] : INFINITY;
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
  return 0;
}

// wgmma inference layout (mlp_tc.cuh) of a 64-wide net: hi | lo TF32 planes of W1 (k padded to 8) and W2, then fp32
// W3, b1, b2, b3 (offsets in floats)
TcNet make_tc_net(const NetL& L) {
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
  return T;
}

// What batched inference of one net needs besides its parameters.
struct InferTarget {
  const KParams& kp;      // net layouts (pol / val), hidden width, smem carve, action squash
  int device, sm_count, max_smem;
  float* blob;            // mma.sync kernel: packed weights (kp.w_floats floats)
  DevBuf& xbuf;           // wide nets: observation tiles
  DevBuf& blob_tc;        // wgmma kernel: packed weight planes
};

// wgmma inference (mlp_tc.cuh).  GOPS_B200_INFER=tc|mma forces one of the two 64-wide paths.
bool infer_use_tc(const InferTarget& t, int64_t batch, const NetL& L) {
  if (t.kp.hid != 64) return false;
  const char* e = getenv("GOPS_B200_INFER");
  if (e && !strcmp(e, "mma")) return false;
  // the wgmma inference kernel keeps the input planes in shared memory: wide inputs stay on the mma.sync kernel
  // whatever the batch size is (no batch-dependent failure)
  if (tc_infer_smem_bytes(make_tc_net(L), 1) > (size_t)t.max_smem) return false;
  if (e && !strcmp(e, "tc")) return true;
  return batch >= 4096;
}

int infer_tc(const InferTarget& t, const float* params, const NetL& L, const float* obs, int64_t batch, float virtual_t,
             float* out, cudaStream_t st, bool squash) {
  TcNet T = make_tc_net(L);
  T.squash = squash ? 1 : 0;
  for (int j = 0; j < MAXA; ++j) { T.half[j] = t.kp.pol_half[j]; T.mid[j] = t.kp.pol_mid[j]; }
  const int wgs = tc_infer_smem_bytes(T, 2) <= (size_t)t.max_smem ? 2 : 1;
  const size_t smem = tc_infer_smem_bytes(T, wgs);
  if (smem > (size_t)t.max_smem) return fail("wgmma inference: input width does not fit in shared memory");
  if (t.blob_tc.ensure(T.blob)) return 1;
  pack_params_tc_kernel<<<8, 256, 0, st>>>(params, T, t.blob_tc.p);
  ++g_launches;
  if (launched("launch#tc-pack")) return 1;
  if (allow_smem((const void*)mlp_infer_tc_kernel<1>, t.device, t.max_smem) ||
      allow_smem((const void*)mlp_infer_tc_kernel<2>, t.device, t.max_smem))
    return 1;
  const long long tiles = (batch + TC_TILE - 1) / TC_TILE;
  const long long ctas = (tiles + wgs - 1) / wgs;
  const int grid = (int)(ctas < t.sm_count ? ctas : t.sm_count);
  if (wgs == 2) mlp_infer_tc_kernel<2><<<grid, 256, smem, st>>>(T, t.blob_tc.p, obs, batch, virtual_t, out);
  else mlp_infer_tc_kernel<1><<<grid, 128, smem, st>>>(T, t.blob_tc.p, obs, batch, virtual_t, out);
  ++g_launches;
  return launched("launch#tc-infer");
}

template <int HH, int SS, int NN>
int launch_infer(const InferTarget& t, const KParams& kp, int grid, size_t smem, int use_val, const float* obs,
                 int64_t batch, float virtual_t, bool squash, float* out, cudaStream_t st) {
  if (allow_smem((const void*)mlp_infer_kernel<HH, SS, NN>, t.device, t.max_smem)) return 1;
  mlp_infer_kernel<HH, SS, NN><<<grid, NN, smem, st>>>(kp, t.blob, use_val, obs, batch, virtual_t, squash ? 1 : 0, out);
  ++g_launches;
  return launched("launch#4");
}

int infer_common(const InferTarget& t, const float* params, int use_val, const float* obs, int64_t batch,
                 float virtual_t, float* out, cudaStream_t st, bool squash) {
  const NetL& L = use_val ? t.kp.val : t.kp.pol;
  if (infer_use_tc(t, batch, L)) return infer_tc(t, params, L, obs, batch, virtual_t, out, st, squash);
  pack_params_kernel<<<t.kp.hid > 64 ? 64 : 8, 256, 0, st>>>(params, L, t.kp.hid, t.blob);
  ++g_launches;
  if (launched("launch#1")) return 1;
  const int cfg = pick_config(t.kp, t.sm_count, t.max_smem, batch, true);
  if (cfg < 0) return fail("no kernel configuration fits in shared memory");
  const int NTc = config_of(t.kp.hid, cfg).NT;
  const long long tiles = (batch + NTc - 1) / NTc;
  const int grid = (int)(tiles < t.sm_count ? tiles : t.sm_count);
  const size_t smem = infer_smem_bytes(t.kp, config_of(t.kp.hid, cfg).S, NTc);
  if (t.kp.hid > 64) {
    if (t.xbuf.ensure((size_t)t.sm_count * t.kp.inp_max * (NTc + 4), true)) return 1;
    KParams kp = t.kp;
    kp.xbuf = t.xbuf.p;
    return launch_infer<256, 32, 256>(t, kp, grid, smem, use_val, obs, batch, virtual_t, squash, out, st);
  }
  if (cfg == 0) return launch_infer<64, 128, 512>(t, t.kp, grid, smem, use_val, obs, batch, virtual_t, squash, out, st);
  if (cfg == 1) return launch_infer<64, 64, 256>(t, t.kp, grid, smem, use_val, obs, batch, virtual_t, squash, out, st);
  return launch_infer<64, 32, 128>(t, t.kp, grid, smem, use_val, obs, batch, virtual_t, squash, out, st);
}

int plan_infer(gops_b200_plan* pl, const float* params, int use_val, const float* obs, int64_t batch, float virtual_t,
               float* out, void* stream, bool squash) {
  if (!pl || !params || !obs || !out) return fail("null argument");
  if (batch <= 0) return fail("empty batch");
  DevGuard dg(pl->device);
  const InferTarget t{pl->kp, pl->device, pl->sm_count, pl->max_smem, use_val ? pl->blob_val.p : pl->blob_pol.p,
                      pl->xbuf, pl->blob_tc};
  return infer_common(t, params, use_val, obs, batch, virtual_t, out, (cudaStream_t)stream, squash);
}

}  // namespace

extern "C" {

int gops_b200_version(void) { return GOPS_B200_ABI_VERSION; }
int64_t gops_b200_launch_count(void) { return (int64_t)g_launches.load(); }
const char* gops_b200_last_error(void) { return last_error(); }

int gops_b200_plan_create(const gops_b200_plan_desc* d, gops_b200_plan** out) {
  ENTRY();
  if (!d || !out) return fail("null argument");
  *out = nullptr;
  KParams kp;
  if (plan_constants(d, kp)) return 1;
  std::unique_ptr<gops_b200_plan> pl(new (std::nothrow) gops_b200_plan());
  if (!pl) return fail("out of host memory");
  pl->desc = *d;
  pl->kp = kp;
  cudaError_t e = cudaGetDevice(&pl->device);
  cudaDeviceProp prop;
  if (e == cudaSuccess) e = cudaGetDeviceProperties(&prop, pl->device);
  if (e != cudaSuccess) return fail(std::string("no CUDA device: ") + cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0) return fail("gops_b200 is built for sm_90a and needs an H100-class (sm_90) device");
  pl->sm_count = prop.multiProcessorCount;
  pl->max_smem = (int)prop.sharedMemPerBlockOptin;

  std::vector<float> gp(d->horizon + 1);
  for (int k = 0; k <= d->horizon; ++k) gp[k] = (float)pow((double)d->gamma, (double)k);
  // note: python evaluates `gamma ** k` on the python float the caller passed; d->gamma is that value
  // rounded to fp32, so callers that need bit parity for non-representable gammas can update gpow via
  // gops_b200_plan_set_gamma (below) with the double value.
  if (pl->gpow.ensure(gp.size()) || pl->blob_pol.ensure(kp.w_floats, true) || pl->blob_val.ensure(kp.w_floats, true) ||
      pl->blob_vtg.ensure(kp.w_floats, true))
    return fail("cudaMalloc failed for plan scratch");
  if (cudaMemcpy(pl->gpow.p, gp.data(), gp.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess)
    return fail("cudaMemcpy(gpow) failed");
  if (kp.obs_scaling) {
    const int od = d->policy.in_dim;
    if (pl->osc.ensure(2 * od)) return fail("cudaMalloc failed");
    if (cudaMemcpy(pl->osc.p, d->obs_scale, od * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(pl->osc.p + od, d->obs_shift, od * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess)
      return fail("cudaMemcpy(obs scale/shift) failed");
    pl->kp.osc = pl->osc.p;
    pl->kp.osh = pl->osc.p + od;
  }
  // wgmma rollout kernel: 64-wide nets whose inputs fit one 16-wide K block, state == obs models
  const bool infadp = d->alg != GOPS_ALG_FHADP;
  if (kp.hid == 64 && kp.pol.in <= tcf::K1 && (!infadp || kp.val.in <= tcf::K1) && kernels_of(d->model)->tc[0][d->alg]) {
    make_net_tcf(kp.pol, pl->pol_tcf);
    if (infadp) make_net_tcf(kp.val, pl->val_tcf); else pl->val_tcf = pl->pol_tcf;
    pl->w_floats_tcf = pl->pol_tcf.blob > pl->val_tcf.blob ? pl->pol_tcf.blob : pl->val_tcf.blob;
    if (pl->blob_pol_tcf.ensure(pl->w_floats_tcf, true) || pl->blob_val_tcf.ensure(pl->w_floats_tcf, true) ||
        pl->blob_vtg_tcf.ensure(pl->w_floats_tcf, true))
      return fail("cudaMalloc failed for plan scratch (wgmma rollout blobs)");
    pl->tc_ok = true;
  }
  pl->kp.gpow = pl->gpow.p;
  pl->kp.blob_pol = pl->blob_pol.p; pl->kp.blob_val = pl->blob_val.p; pl->kp.blob_vtg = pl->blob_vtg.p;
  *out = pl.release();
  return 0;
}

int gops_b200_plan_set_gamma(gops_b200_plan* pl, double gamma) {
  if (!pl) return fail("null plan");
  DevGuard dg(pl->device);
  std::vector<float> gp(pl->kp.horizon + 1);
  for (int k = 0; k <= pl->kp.horizon; ++k) gp[k] = (float)pow(gamma, (double)k);
  pl->kp.gamma = (float)gamma;
  CUDA_OK(cudaMemcpy(pl->gpow.p, gp.data(), gp.size() * sizeof(float), cudaMemcpyHostToDevice));
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
  if (path == GOPS_PATH_TC && !pl->tc_ok && !layerwise_built(pl))
    return fail("the wgmma rollout kernel is not built for this plan (needs 64-wide nets, <= 16 inputs, idpendulum / lq)");
  pl->path = path;
  return 0;
}
int gops_b200_plan_last_path(const gops_b200_plan* pl) { return pl ? pl->last_path : -1; }

int gops_b200_plan_set_constraint(gops_b200_plan* pl, int mode, float coef) {
  if (!pl) return fail("null plan");
  if (mode < 0 || mode > 4) return fail("unknown constraint mode");
  if (mode == 4) {
    // SPIL runs on the mma.sync / FFMA rollout kernel only
    if (!(pl->desc.model == GOPS_MODEL_VEH3DOFCONTI && pl->desc.veh_errcstr) && pl->desc.model != GOPS_MODEL_MOBILEROBOT)
      return fail("the SPIL constraint mode is built for pyth_veh3dofconti_errcstr and pyth_mobilerobot only");
    if (pl->desc.alg != GOPS_ALG_FHADP && pl->desc.alg != GOPS_ALG_INFADP_VALUE)
      return fail("the SPIL constraint mode needs an FHADP (policy) or INFADP_VALUE (value) plan");
    if (pl->desc.open_loop || pl->tc_ok || layerwise_built(pl))
      return fail("the SPIL constraint mode is not built for the wgmma or layer-wise rollout paths");
    pl->kp.cstr_mode = mode;
    pl->kp.cstr_coef = 1.f;
    return 0;
  }
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

int gops_b200_plan_set_spil_weights(gops_b200_plan* pl, const float* weights) {
  if (!pl) return fail("null plan");
  pl->kp.spil_w = weights;
  return 0;
}

int gops_b200_plan_set_model_io(gops_b200_plan* pl, const float* noise, float* constraint_out) {
  if (!pl) return fail("null plan");
  if (pl->desc.model != GOPS_MODEL_MOBILEROBOT) return fail("plan_set_model_io: this env model takes no noise");
  pl->kp.noise = noise;
  pl->kp.cstr_out = constraint_out;
  return 0;
}

int gops_b200_spil_controller(const float* tail, int64_t batch_global, double kp, double ki, double kd,
                              double chance_thre0, double chance_thre1, double* state, float* weights, void* stream) {
  ENTRY();
  if (!tail || !state || !weights) return fail("null argument");
  if (batch_global <= 0) return fail("empty batch");
  const int dev = device_of(state);
  if (dev < 0 || dev >= kMaxDevices) return fail("device index out of range");
  DevGuard dg(dev);
  spil_controller_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(tail, (long long)batch_global, kp, ki, (float)kd,
                                                             chance_thre0, chance_thre1, state, weights);
  ++g_launches;
  return launched("launch#spil-controller");
}

int gops_b200_plan_launch_info(const gops_b200_plan* pl, int32_t* out4) {
  if (!pl || !out4) return fail("null argument");
  out4[0] = pl->last_grid; out4[1] = pl->last_NT; out4[2] = pl->last_S; out4[3] = (int32_t)pl->last_smem;
  return 0;
}

int gops_b200_plan_destroy(gops_b200_plan* pl) {
  ENTRY();
  if (!pl) return 0;
  DevGuard dg(pl->device);
  if (getenv("GOPS_B200_DEBUG"))
    fprintf(stderr, "[gops_b200] destroy plan %p alg %d model %d\n", (void*)pl, pl->desc.alg, pl->desc.model);
  if (pl->ev0) { cudaEventDestroy(pl->ev0); cudaEventDestroy(pl->ev1); }
  if (pl->lw_exec) cudaGraphExecDestroy(pl->lw_exec);
  if (pl->lw_cap_stream) cudaStreamDestroy(pl->lw_cap_stream);
  if (pl->lw_net) gops_b200_mlpnet_destroy(pl->lw_net);
  delete pl;    // frees the device buffers
  return 0;
}

int64_t gops_b200_plan_param_count(const gops_b200_plan* pl, int which) {
  if (!pl) return -1;
  return which == 0 ? pl->kp.pol.nparam : pl->kp.val.nparam;
}

int gops_b200_rollout_grad(gops_b200_plan* pl, const gops_b200_batch* b, const float* policy_params,
                           const float* value_params, const float* vtarget_params, float inv_batch_global,
                           float* grad_out, float* scalars_out, void* stream) {
  ENTRY();
  if (!pl || !policy_params || !grad_out || !scalars_out) return fail("null argument");
  const int alg = pl->desc.alg;
  if (alg != GOPS_ALG_FHADP && !vtarget_params) return fail("vtarget_params required for INFADP");
  if (alg == GOPS_ALG_INFADP_VALUE && !value_params) return fail("value_params required for INFADP value update");
  const Route route = b ? rollout_route(pl, alg, b->batch) : Route::Mma;
  if (check_batch(pl, b, route == Route::Layerwise)) return 1;
  DevGuard dg(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  KParams p = bind_batch(pl, b, alg);
  p.inv_B = inv_batch_global;
  if (p.cstr_mode == 4) {
    if (route != Route::Mma) return fail("the SPIL constraint mode runs on the mma.sync rollout kernel only");
    if (alg == GOPS_ALG_FHADP && !p.spil_w) return fail("SPIL policy pass: weights pointer not set (plan_set_spil_weights)");
  }
  if (route == Route::Layerwise) return launch_layerwise(pl, p, policy_params, st, grad_out, scalars_out);
  if (launch_pack(pl, route, policy_params, false, pl->blob_pol.p, pl->blob_pol_tcf.p, st)) return 1;
  if (alg != GOPS_ALG_FHADP && launch_pack(pl, route, vtarget_params, true, pl->blob_vtg.p, pl->blob_vtg_tcf.p, st)) return 1;
  if (alg == GOPS_ALG_INFADP_VALUE && launch_pack(pl, route, value_params, true, pl->blob_val.p, pl->blob_val_tcf.p, st))
    return 1;
  return launch_fused(pl, p, route, st, grad_out, scalars_out);
}

int gops_b200_rollout_trace(gops_b200_plan* pl, const gops_b200_batch* b, const float* policy_params, float* obs_out,
                            float* act_out, float* rew_out, float* done_out, void* stream) {
  ENTRY();
  if (!pl || !policy_params) return fail("null argument");
  if (check_batch(pl, b, false)) return 1;
  const Route route = rollout_route(pl, ALG_TRACE, b->batch);
  DevGuard dg(pl->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (launch_pack(pl, route, policy_params, false, pl->blob_pol.p, pl->blob_pol_tcf.p, st)) return 1;
  KParams p = bind_batch(pl, b, ALG_TRACE);
  p.inv_B = 1.f;
  p.tr_obs = obs_out; p.tr_act = act_out; p.tr_rew = rew_out; p.tr_done = done_out;
  return launch_fused(pl, p, route, st, nullptr, nullptr);
}

int gops_b200_policy_forward(gops_b200_plan* pl, const float* policy_params, const float* obs, int64_t batch,
                             float virtual_t, float* act_out, void* stream) {
  return plan_infer(pl, policy_params, 0, obs, batch, virtual_t, act_out, stream, true);
}

int gops_b200_value_forward(gops_b200_plan* pl, const float* value_params, const float* obs, int64_t batch,
                            float* v_out, void* stream) {
  if (pl && pl->desc.alg == GOPS_ALG_FHADP) return fail("plan has no value network");
  return plan_infer(pl, value_params, 1, obs, batch, 0.f, v_out, stream, false);
}

int gops_b200_mlp_forward(const gops_b200_mlp_desc* net, const float* params, const float* obs, int64_t batch,
                          float virtual_t, const float* act_low, const float* act_high, float* out, void* stream) {
  ENTRY();
  if (!net || !params || !obs || !out) return fail("null argument");
  if (batch <= 0) return fail("empty batch");
  const int dev = device_of(params);
  if (dev < 0 || dev >= kMaxDevices) return fail("device index out of range");
  DevGuard dg(dev);
  struct Scratch { DevBuf blob, xbuf, blob_tc; };
  static thread_local Scratch scratch_of[kMaxDevices];   // reusable staging buffers per host thread and device
  Scratch& s = scratch_of[dev];
  KParams kp;
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
  if (s.blob.ensure(kp.w_floats)) return 1;
  const InferTarget t{kp, dev, prop.multiProcessorCount, (int)prop.sharedMemPerBlockOptin, s.blob.p, s.xbuf, s.blob_tc};
  return infer_common(t, params, 0, obs, batch, virtual_t, out, (cudaStream_t)stream, act_low != nullptr);
}

int gops_b200_model_step(gops_b200_plan* pl, const gops_b200_batch* b, const float* action, float* next_obs,
                         float* reward, float* next_done, float* next_state, float* next_ref_points,
                         float* next_ref_time, void* stream) {
  ENTRY();
  if (!pl || !b || !action || !next_obs || !reward || !next_done) return fail("null argument");
  if (b->batch <= 0 || !b->obs || !b->done) return fail("bad batch");
  DevGuard dg(pl->device);
  const KParams p = bind_batch(pl, b, pl->desc.alg);
  const unsigned grid = (unsigned)((b->batch + 127) / 128);
  cudaStream_t st = (cudaStream_t)stream;
  const int act_dim = pl->desc.policy.out_dim;
  if (pl->desc.model == GOPS_MODEL_VEH3DOFCONTI || pl->desc.model == GOPS_MODEL_VEH3DOF_TRACKING) {
    const bool conti = pl->desc.model == GOPS_MODEL_VEH3DOFCONTI;
    if (!b->state || !next_state) return fail("model_step: vehicle models need state and next_state");
    if (conti && (!b->ref_points || !b->path_num || !b->u_num || !b->ref_time || !next_ref_points || !next_ref_time))
      return fail("model_step: pyth_veh3dofconti needs ref_points, path_num, u_num, ref_time and their outputs");
    if (!conti && (!b->reference || b->ref_t < 0 || b->ref_t + p.veh_P + 2 > b->ref_len))
      return fail("model_step: veh3dof_tracking reference too short for t + 1 + pre_horizon + 1 points");
    if (pl->desc.veh_detour && (!b->surr || b->ref_t + 2 > b->surr_len))
      return fail("model_step: veh3dof_tracking_detour needs the surrounding-vehicle predictions for t and t + 1");
    if (pl->desc.veh_detour) launch_veh_step_detour(p, action, next_obs, reward, next_done, next_state, st);
    else if (conti) veh_step_kernel<1><<<grid, 128, 0, st>>>(p, action, next_obs, reward, next_done, next_state,
                                                        next_ref_points, next_ref_time);
    else veh_step_kernel<2><<<grid, 128, 0, st>>>(p, action, next_obs, reward, next_done, next_state,
                                                  next_ref_points, next_ref_time);
    ++g_launches;
    return launched("veh_step launch");
  }
  if (pl->desc.model == GOPS_MODEL_MOBILEROBOT && !p.noise)
    return fail("model_step: pyth_mobilerobot needs its obstacle noise [batch][2] (gops_b200_plan_set_model_io)");
  StepFn fn = kernels_of(pl->desc.model)->step;
  if (!fn) return fail("model_step: env model kind not built into this library");
  fn<<<grid, 128, 0, st>>>(p, action, act_dim, next_obs, reward, next_done);
  ++g_launches;
  return launched("launch#5");
}

int gops_b200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                        int32_t step, double lr, double beta1, double beta2, double eps, void* stream) {
  ENTRY();
  if (!params || !grads || !exp_avg || !exp_avg_sq) return fail("null argument");
  if (n <= 0 || step < 1) return fail("bad n/step");
  DevGuard dg(params);
  // python-side scalars of torch/optim/adam.py are doubles; only the tensor math is fp32
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  const float step_size = (float)(lr / bc1);
  const float bc2_sqrt = (float)sqrt(bc2);
  adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      params, grads, exp_avg, exp_avg_sq, n, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps,
      step_size, bc2_sqrt);
  ++g_launches;
  return launched("launch#6");
}

int gops_b200_polyak(float* target, const float* src, float tau, int64_t n, void* stream) {
  ENTRY();
  if (!target || !src || n <= 0) return fail("bad argument");
  DevGuard dg(target);
  polyak_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(target, src, tau, n);
  ++g_launches;
  return launched("launch#7");
}

}  // extern "C"
