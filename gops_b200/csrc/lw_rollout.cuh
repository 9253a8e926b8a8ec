// Layer-wise FHADP rollout for nets that do not fit the fused kernels (hidden width 256): the horizon unroll of
// gops/algorithm/fhadp.py:113-125 as per-step kernels around the wgmma dense layers of dense_tc.cuh.
//
//   forward step k :  policy MLP on X_k (3 wgmma GEMMs, activations kept in slot k)  ->  z_k
//                     lw_step_kernel: tanh squash / wrapper chain / env-model step -> state_{k+1}, done_{k+1}, X_{k+1}, reward
//   reverse step k :  lw_reverse_kernel: finish lambda_{k+1} with the observation adjoint of step k + 1's input
//                     gradient, then the hand-derived adjoint of step k  ->  zbar_k, lambda_k (partial)
//                     policy MLP backward of slot k (wgmma dgrad GEMMs; deltas kept)  ->  dX_k
//   weight gradients: ONE contraction per layer over all H x B rows (gops_b200_mlpnet_wgrad_slots).
// The per-sample arithmetic is the fused kernels' own: the wrapper chain, the model steps, the vehicle rewards and their
// adjoints are the device functions of models.cuh / models_veh.cuh, one thread per sample;
// states live in HBM between the steps: 0.5 GB of activations per update for C3 (8192 x 60 x [256 + 256 + 248] fp32 x2),
// 0.1 ms of HBM time -- the path stays tensor / launch bound.
#pragma once
#include "models.cuh"

namespace gops {

struct LwArgs {
  int k, ldx, act_dim;
  long long bstride;       // rows between consecutive steps in X
  long long zs_k, zs_b;    // Z / Zb strides (floats) per step and per sample: closed loop [H][rows][A] -> (rows A, A);
                           // open loop (FHADP2: one policy call emits all H actions) [B][H A] -> (A, H A)
  float* S;                // [H + 1][NS][B] states (SoA)
  float* Dn;               // [H + 1][B] done flags
  float* X;                // [H + 1][bstride][ldx] policy inputs (observation + time column); nullptr: open loop
  const float* Z;          // [H][bstride][act_dim] policy pre-activations
  float* Zb;               // [H][bstride][act_dim] their adjoints
  float* lam;              // [NS][B] adjoint of the state entering the next reverse step
  const float* dX;         // [bstride][ldx] input gradient of step k + 1 (reverse) or nullptr
  float* vacc;             // [B] discounted reward sums
  float* cacc;             // detour: [3][B] discounted constraint sums (exterior or Lagrangian | interior log) and the infeasible flag
  float* xcar;             // detour: [B][ldx] adjoint handed back by frozen copies of an observation row
};

// copy the caller's batch into step 0: X_0 = [obs | time 1], S_0, Dn_0
template <class M>
__global__ void lw_init_kernel(const __grid_constant__ KParams p, const __grid_constant__ LwArgs a) {
  constexpr int NS = M::NS;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long B = p.batch;
  if (b >= B) return;
  const int obs_dim = p.pol.obs;
  if (a.X != nullptr) {
    float* x = a.X + b * a.ldx;
    for (int f = 0; f < obs_dim; ++f) x[f] = p.obs[b * obs_dim + f];
    if (p.pol.time_input) x[obs_dim] = 1.f;
    for (int f = obs_dim + p.pol.time_input; f < a.ldx; ++f) x[f] = 0.f;
  }
#pragma unroll
  for (int f = 0; f < NS; ++f) {
    float v = 0.f;
    if (M::KIND == 0) v = f < obs_dim ? p.obs[b * obs_dim + f] : 0.f;
    else v = f < 6 ? p.state[b * 6 + f] : 0.f;
    a.S[(size_t)f * B + b] = v;
  }
  a.Dn[b] = p.done[b] != 0.f ? 1.f : 0.f;
  a.vacc[b] = 0.f;
#pragma unroll
  for (int f = 0; f < NS; ++f) a.lam[(size_t)f * B + b] = 0.f;
}

// forward step k (reference: one iteration of the loop in fhadp.py:118-123 through the wrapper chain).
// SUB threads per sample: all of them run the (cheap) action / reward / state update redundantly, the observation
// rebuild -- P + 1 ego-frame transforms per sample, the bulk of the work for the vehicle models -- is dealt over them.
constexpr int LW_SUB = 8;
template <class M>
__global__ void lw_step_kernel(const __grid_constant__ KParams p, const __grid_constant__ LwArgs a) {
  constexpr int NS = M::NS;
  constexpr int SUB = M::KIND == 0 ? 1 : LW_SUB;
  const long long gt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long b = gt / SUB;
  const int sub = (int)(gt % SUB);
  const long long B = p.batch;
  if (b >= B) return;
  const int k = a.k, obs_dim = p.pol.obs;
  const float* Sk = a.S + (size_t)k * NS * B;
  float* Sn = a.S + (size_t)(k + 1) * NS * B;
  float st[NS], z[MAXA], act[MAXA], g[MAXA];
#pragma unroll
  for (int f = 0; f < NS; ++f) st[f] = Sk[(size_t)f * B + b];
  bool dn = a.Dn[(size_t)k * B + b] != 0.f;
#pragma unroll
  for (int j = 0; j < MAXA; ++j) z[j] = j < a.act_dim ? a.Z[(size_t)k * a.zs_k + (size_t)b * a.zs_b + j] : 0.f;
  process_action(p, a.act_dim, z, act, g, nullptr);
  const bool active = p.mask_at_done ? !dn : true;
  const bool wx = a.X != nullptr;
  const float* xk = wx ? a.X + ((size_t)k * a.bstride + b) * a.ldx : nullptr;
  float* xn = wx ? a.X + ((size_t)(k + 1) * a.bstride + b) * a.ldx : nullptr;      // the caller allocates H + 1 input slabs
  float r = 0.f;
  if constexpr (M::KIND == 0) {
    wrapped_step<M>(p, obs_dim, st, act, active, r, dn);
#pragma unroll
    for (int f = 0; f < NS; ++f)
      if (wx && f < obs_dim) xn[f] = st[f];
  } else {
    if (active) {
      const VehC vc = veh_const();
      RefWindow<2, 1> w;
      w.base = p.reference + (size_t)b * p.ref_len * 4;
      float q[4];
      w.k0 = p.ref_t + k;
      w.get(0, q);
      r = M::reward(st, q, act);
      veh_step(vc, st, act);
      w.k0 = p.ref_t + k + 1;
      if (wx) {      // get_obs of the new state: point i of the window by sub-thread i mod SUB
        float sn, cs, o4[4];
        sincosf(-st[2], &sn, &cs);
        for (int i = sub; i <= p.veh_P; i += SUB) {
          w.get(i, q);
          ego_obs(st, cs, sn, q[0], q[1], q[2], q[3], o4);
          const int f0 = i == 0 ? 0 : 6 + 4 * (i - 1);
#pragma unroll
          for (int c = 0; c < 4; ++c) xn[f0 + c] = to_outer(p, f0 + c, o4[c]);
          if (i == 0) {
            xn[4] = to_outer(p, 4, st[4]);
            xn[5] = to_outer(p, 5, st[5]);
          }
        }
      }
      w.get(0, q);
      dn = M::done(st, q);
    } else if (wx) {
      for (int f = sub; f < obs_dim; f += SUB) xn[f] = xk[f];        // MaskAtDone: the observation is frozen
    }
  }
  if (sub != 0) return;
  if (wx) {
    if (p.pol.time_input) xn[obs_dim] = (float)(k + 2);
    for (int f = obs_dim + p.pol.time_input; f < a.ldx; ++f) xn[f] = 0.f;
  }
  r = shape_reward(p, r);
  a.vacc[b] += r * p.gpow[k];
#pragma unroll
  for (int f = 0; f < NS; ++f) Sn[(size_t)f * B + b] = st[f];
  a.Dn[(size_t)(k + 1) * B + b] = dn ? 1.f : 0.f;
}

// reverse step k: lambda_{k+1} += Obs^T dX_{k+1} (if a.dX), then the adjoint of step k -> Zb_k, lambda (in place)
template <class M>
__global__ void lw_reverse_kernel(const __grid_constant__ KParams p, const __grid_constant__ LwArgs a) {
  constexpr int NS = M::NS;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long B = p.batch;
  if (b >= B) return;
  const int k = a.k, obs_dim = p.pol.obs;
  float lam[NS], st[NS];
#pragma unroll
  for (int f = 0; f < NS; ++f) lam[f] = a.lam[(size_t)f * B + b];
  if (a.dX != nullptr) {             // finish lambda_{k+1}: the policy path of step k + 1 (sample must have been live there)
    const bool live = p.mask_at_done ? a.Dn[(size_t)(k + 1) * B + b] == 0.f : true;
    if (live) {
      const float* dx = a.dX + (size_t)b * a.ldx;
      if constexpr (M::KIND == 0) {
#pragma unroll
        for (int f = 0; f < NS; ++f)
          if (f < obs_dim) lam[f] += dx[f];
      } else {
        const float* S1 = a.S + (size_t)(k + 1) * NS * B;
        float s1[NS];
#pragma unroll
        for (int f = 0; f < NS; ++f) s1[f] = S1[(size_t)f * B + b];
        RefWindow<2, 1> w;
        w.base = p.reference + (size_t)b * p.ref_len * 4;
        w.k0 = p.ref_t + k + 1;
        const float zero6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        veh_obs_bwd<2, 1>(s1, w, p.veh_P, dx, 1, zero6, p.obs_scaling ? p.osc : nullptr, lam);
      }
    }
  }
  const float* Sk = a.S + (size_t)k * NS * B;
#pragma unroll
  for (int f = 0; f < NS; ++f) st[f] = Sk[(size_t)f * B + b];
  const bool dnk = a.Dn[(size_t)k * B + b] != 0.f;
  const bool active = p.mask_at_done ? !dnk : true;
  float zb[MAXA];
#pragma unroll
  for (int j = 0; j < MAXA; ++j) zb[j] = 0.f;
  if (active) {
    float z[MAXA], act[MAXA], g[MAXA], abar[MAXA];
#pragma unroll
    for (int j = 0; j < MAXA; ++j) z[j] = j < a.act_dim ? a.Z[(size_t)k * a.zs_k + (size_t)b * a.zs_b + j] : 0.f;
    process_action(p, a.act_dim, z, act, g, nullptr);
    const float rho = reward_adjoint(p, k);
#pragma unroll
    for (int j = 0; j < MAXA; ++j) abar[j] = 0.f;
    if constexpr (M::KIND == 0) {
      wrapped_step_bwd<M>(p, obs_dim, st, act, rho, lam, abar);
    } else {
      const VehC vc = veh_const();
      veh_step_bwd(vc, st, act, lam, abar);
      RefWindow<2, 1> w;
      w.base = p.reference + (size_t)b * p.ref_len * 4;
      w.k0 = p.ref_t + k;
      float q[4];
      w.get(0, q);
      M::reward_bwd(st, q, act, rho, lam, abar);
    }
#pragma unroll
    for (int j = 0; j < MAXA; ++j) zb[j] = abar[j] * g[j];
  }
#pragma unroll
  for (int j = 0; j < MAXA; ++j)
    if (j < a.act_dim) a.Zb[(size_t)k * a.zs_k + (size_t)b * a.zs_b + j] = zb[j];
#pragma unroll
  for (int f = 0; f < NS; ++f) a.lam[(size_t)f * B + b] = lam[f];
}

// loss / #done partial sums in fixed order: block partials, then one thread
static __global__ void lw_scalars_kernel(const float* __restrict__ vacc, const float* __restrict__ dn_last, long long B, float inv_B,
                                  float* __restrict__ partial) {
  __shared__ float s0[256], s1[256];
  float a = 0.f, d = 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < B; i += (long long)gridDim.x * 256) {
    a += -vacc[i] * inv_B;
    d += dn_last[i];
  }
  s0[threadIdx.x] = a; s1[threadIdx.x] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    float x = 0.f, y = 0.f;
    for (int i = 0; i < 256; ++i) { x += s0[i]; y += s1[i]; }
    partial[2 * blockIdx.x] = x; partial[2 * blockIdx.x + 1] = y;
  }
}
static __global__ void lw_scalars_final_kernel(const float* __restrict__ partial, int nb, float* __restrict__ scalars) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float x = 0.f, y = 0.f;
    for (int i = 0; i < nb; ++i) { x += partial[2 * i]; y += partial[2 * i + 1]; }
    scalars[0] = x; scalars[1] = 0.f; scalars[2] = y; scalars[3] = 0.f;
  }
}

typedef void (*LwFn)(const KParams, const LwArgs);

}  // namespace gops
