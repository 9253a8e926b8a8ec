// env_gen_ocp veh3dof_tracking_detour / veh3dof_tracking_surrcstr on the layer-wise path (lw_rollout.cuh): the tracking
// model plus ONE surrounding vehicle (reference: gops/env/env_gen_ocp/env_model/veh3dof_tracking_detour_model.py:13-176,
// veh3dof_tracking_surrcstr_model.py:13-181 -- same structure, other circle radius / reward / bound; EnvModel.forward
// env_model/pyth_base_model.py:109-119, MaskAtDone wrapper/mask_at_done.py:26-40) and the constrained FHADP variants on
// it (fhadp_exterior.py:55-70, fhadp_lagrangian.py:59-71, fhadp_interior.py:55-84).
//
// What differs from the plain tracking model:
//   * four more observation entries: the surrounding vehicle's pose in the ego frame and its raw speed (:62-76);
//   * reward weights, the +2 offset and the lateral termination bound (:133-163);
//   * info["constraint"] = 2 r - min distance between the two circles of each vehicle, of the INCOMING state (:78-131);
//   * the constraint is read every step, also after `done`: MaskAtDone freezes the observation and zeroes the reward,
//     but info["state"] keeps evolving under the actions the policy emits for the frozen observation.  So the state is
//     stepped unconditionally, a frozen row X_{k+1} = X_k hands its adjoint back to X_k (`xcar`), and only a row that was
//     produced by get_obs pushes its adjoint onto the state.
#pragma once
#include "lw_rollout.cuh"

namespace gops {

constexpr float DETOUR_EPS = 1e-8f;        // fhadp_interior.py:19 EPSILON

// surrounding vehicle k of sample b: [x, y, phi, u, delta]
__device__ __forceinline__ const float* detour_surr(const KParams& p, long long b, int k) {
  return p.surr + ((size_t)b * p.surr_len + (size_t)(p.ref_t + k)) * 5;
}

// c = 2 r - min_{i,j} |ego circle i - surrounding circle j|;  g = dc / d(x, y, phi)
__device__ __forceinline__ float detour_constraint(const KParams& p, const float* s, const float* q, float* g) {
  const float d = p.veh_dc;
  float sn, cs, qs, qc;
  sincosf(s[2], &sn, &cs);
  sincosf(q[2], &qs, &qc);
  float best = 3.402823466e+38f, bux = 0.f, buy = 0.f, bsg = 1.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float sg = i == 0 ? 1.f : -1.f;
    const float ex = s[0] + sg * d * cs, ey = s[1] + sg * d * sn;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float tg = j == 0 ? 1.f : -1.f;
      const float dx = ex - (q[0] + tg * d * qc), dy = ey - (q[1] + tg * d * qs);
      const float dist = sqrtf(dx * dx + dy * dy);
      if (dist < best) { best = dist; bux = dx / dist; buy = dy / dist; bsg = sg; }
    }
  }
  if (g != nullptr) {
    g[0] = -bux;
    g[1] = -buy;
    g[2] = -(bux * (-bsg * d * sn) + buy * (bsg * d * cs));
  }
  return p.veh_2r - best;
}

// forward step k
__global__ void lw_step_detour_kernel(const __grid_constant__ KParams p, const __grid_constant__ LwArgs a) {
  constexpr int NS = 6, SUB = LW_SUB;
  const long long gt = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long b = gt / SUB;
  const int sub = (int)(gt % SUB);
  const long long B = p.batch;
  if (b >= B) return;
  const int k = a.k, obs_dim = p.pol.obs, P = p.veh_P;
  const float* Sk = a.S + (size_t)k * NS * B;
  float* Sn = a.S + (size_t)(k + 1) * NS * B;
  float st[NS], z[MAXA], act[MAXA], g[MAXA];
#pragma unroll
  for (int f = 0; f < NS; ++f) st[f] = Sk[(size_t)f * B + b];
  const bool dn = a.Dn[(size_t)k * B + b] != 0.f;
  const bool frozen = p.mask_at_done && dn;
#pragma unroll
  for (int j = 0; j < MAXA; ++j) z[j] = j < a.act_dim ? a.Z[(size_t)k * a.zs_k + (size_t)b * a.zs_b + j] : 0.f;
  process_action(p, a.act_dim, z, act, g, nullptr);
  const float* xk = a.X + ((size_t)k * a.bstride + b) * a.ldx;
  float* xn = a.X + ((size_t)(k + 1) * a.bstride + b) * a.ldx;
  RefWindow<2, 1> w;
  w.base = p.reference + (size_t)b * p.ref_len * 4;
  float q[4];
  float r = 0.f, c = 0.f;
  if (sub == 0) {
    c = detour_constraint(p, st, detour_surr(p, b, k), nullptr);
    if (!frozen) {
      w.k0 = p.ref_t + k;
      w.get(0, q);
      const float ex = st[0] - q[0], ey = st[1] - q[1], ep = angle_normalize(st[2] - q[2]), eu = st[3] - q[3];
      r = -p.veh_rscale * (p.veh_rc[0] * (ex * ex) + p.veh_rc[1] * (ey * ey) + p.veh_rc[2] * (ep * ep) + p.veh_rc[3] * (eu * eu) +
                           p.veh_rc[4] * (st[5] * st[5]) + p.veh_rc[5] * (act[0] * act[0]) + p.veh_rc[6] * (act[1] * act[1])) +
          p.veh_roff;
    }
  }
  const VehC vc = veh_const();
  veh_step(vc, st, act);                       // info["state"] advances whether or not the sample is done
  w.k0 = p.ref_t + k + 1;
  if (!frozen) {                               // get_obs of the new state; the window points are dealt over the sub-threads
    float sn, cs, o4[4];
    sincosf(-st[2], &sn, &cs);
    for (int i = sub; i <= P + 1; i += SUB) {
      if (i <= P) {
        w.get(i, q);
        ego_obs(st, cs, sn, q[0], q[1], q[2], q[3], o4);
        const int f0 = i == 0 ? 0 : 6 + 4 * (i - 1);
#pragma unroll
        for (int e = 0; e < 4; ++e) xn[f0 + e] = o4[e];
        if (i == 0) { xn[4] = st[4]; xn[5] = st[5]; }
      } else {                                 // the surrounding vehicle: ego-frame pose, raw speed
        const float* sp = detour_surr(p, b, k + 1);
        ego_obs(st, cs, sn, sp[0], sp[1], sp[2], 0.f, o4);
        const int f0 = 6 + 4 * P;
        xn[f0] = o4[0]; xn[f0 + 1] = o4[1]; xn[f0 + 2] = o4[2]; xn[f0 + 3] = sp[3];
      }
    }
  } else {
    for (int f = sub; f < obs_dim; f += SUB) xn[f] = xk[f];      // MaskAtDone: the observation is frozen
  }
  if (sub != 0) return;
  w.get(0, q);
  const bool term = (fabsf(st[0] - q[0]) > 5.f) || (fabsf(st[1] - q[1]) > p.veh_ydone) ||
                    (fabsf(angle_normalize(st[2] - q[2])) > 3.14159265358979323846f);
  if (p.pol.time_input) xn[obs_dim] = (float)(k + 2);
  for (int f = obs_dim + p.pol.time_input; f < a.ldx; ++f) xn[f] = 0.f;
  r = shape_reward(p, r);      // MaskAtDone sits inside ShapingReward (masked r = 0)
  a.vacc[b] += r * p.gpow[k];
  if (p.cstr_mode != 0) {
    const float pos = fmaxf(c, 0.f);
    a.cacc[b] += (p.cstr_mode == 2 ? pos : pos * pos) * p.gpow[k];
    a.cacc[B + b] += logf(-fminf(c, 0.f) + DETOUR_EPS) * p.gpow[k];
    if (!(c < 0.f)) a.cacc[2 * B + b] = 1.f;
  }
#pragma unroll
  for (int f = 0; f < NS; ++f) Sn[(size_t)f * B + b] = st[f];
  a.Dn[(size_t)(k + 1) * B + b] = (dn || term) ? 1.f : 0.f;
}

// reverse step k: route the adjoint of row X_{k+1} (policy input gradient of step k + 1 + what later frozen copies
// handed back), then the adjoint of step k
__global__ void lw_reverse_detour_kernel(const __grid_constant__ KParams p, const __grid_constant__ LwArgs a) {
  constexpr int NS = 6;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long B = p.batch;
  if (b >= B) return;
  const int k = a.k, obs_dim = p.pol.obs, P = p.veh_P;
  float lam[NS], st[NS];
#pragma unroll
  for (int f = 0; f < NS; ++f) lam[f] = a.lam[(size_t)f * B + b];
  const bool dnk = a.Dn[(size_t)k * B + b] != 0.f;
  const bool frozen = p.mask_at_done && dnk;
  float* xc = a.xcar + (size_t)b * a.ldx;
  if (a.dX != nullptr) {                         // k < H - 1: row X_{k+1} fed the policy of step k + 1
    const float* dx = a.dX + (size_t)b * a.ldx;
    if (frozen) {                                // X_{k+1} = X_k: hand everything back to X_k
      for (int f = 0; f < obs_dim; ++f) xc[f] += dx[f];
    } else {                                     // X_{k+1} = get_obs(state_{k+1}, context t + k + 1)
      const float* S1 = a.S + (size_t)(k + 1) * NS * B;
      float s1[NS];
#pragma unroll
      for (int f = 0; f < NS; ++f) s1[f] = S1[(size_t)f * B + b];
      float sn, cs;
      sincosf(-s1[2], &sn, &cs);
      RefWindow<2, 1> w;
      w.base = p.reference + (size_t)b * p.ref_len * 4;
      w.k0 = p.ref_t + k + 1;
      float bx = 0.f, by = 0.f, bphi = 0.f, bu = 0.f;
      for (int i = 0; i <= P + 1; ++i) {
        float q[4];
        const int f0 = i == 0 ? 0 : (i <= P ? 6 + 4 * (i - 1) : 6 + 4 * P);
        if (i <= P) w.get(i, q);
        else { const float* sp = detour_surr(p, b, k + 1); q[0] = sp[0]; q[1] = sp[1]; q[2] = sp[2]; q[3] = 0.f; }
        const float ox = dx[f0] + xc[f0], oy = dx[f0 + 1] + xc[f0 + 1], op = dx[f0 + 2] + xc[f0 + 2];
        const float ou = i <= P ? dx[f0 + 3] + xc[f0 + 3] : 0.f;      // the surrounding speed does not depend on the state
        const float ddx = q[0] - s1[0], ddy = q[1] - s1[1];
        const float vx = ddx * cs - ddy * sn, vy = ddx * sn + ddy * cs;
        bx += -cs * ox - sn * oy;
        by += sn * ox - cs * oy;
        bphi += vy * ox - vx * oy - op;
        bu += -ou;
      }
      lam[0] += bx; lam[1] += by; lam[2] += bphi; lam[3] += bu;
      lam[4] += dx[4] + xc[4];
      lam[5] += dx[5] + xc[5];
      for (int f = 0; f < obs_dim; ++f) xc[f] = 0.f;
    }
  }
  const float* Sk = a.S + (size_t)k * NS * B;
#pragma unroll
  for (int f = 0; f < NS; ++f) st[f] = Sk[(size_t)f * B + b];
  float z[MAXA], act[MAXA], g[MAXA], abar[MAXA];
#pragma unroll
  for (int j = 0; j < MAXA; ++j) z[j] = j < a.act_dim ? a.Z[(size_t)k * a.zs_k + (size_t)b * a.zs_b + j] : 0.f;
  process_action(p, a.act_dim, z, act, g, nullptr);
#pragma unroll
  for (int j = 0; j < MAXA; ++j) abar[j] = 0.f;
  const VehC vc = veh_const();
  veh_step_bwd(vc, st, act, lam, abar);          // the state chain runs through done samples too
  if (!frozen) {                                 // reward of step k (masked once done)
    const float rho = reward_adjoint(p, k);
    const float r2 = -2.f * p.veh_rscale;
    abar[0] += rho * (r2 * p.veh_rc[5] * act[0]);
    abar[1] += rho * (r2 * p.veh_rc[6] * act[1]);
    RefWindow<2, 1> w;
    w.base = p.reference + (size_t)b * p.ref_len * 4;
    w.k0 = p.ref_t + k;
    float q[4];
    w.get(0, q);
    lam[0] += rho * (r2 * p.veh_rc[0] * (st[0] - q[0]));
    lam[1] += rho * (r2 * p.veh_rc[1] * (st[1] - q[1]));
    lam[2] += rho * (r2 * p.veh_rc[2] * angle_normalize(st[2] - q[2]));
    lam[3] += rho * (r2 * p.veh_rc[3] * (st[3] - q[3]));
    lam[5] += rho * (r2 * p.veh_rc[4] * st[5]);
  }
  if (p.cstr_mode != 0) {                        // constraint of the incoming state of step k
    float gc[3];
    const float c = detour_constraint(p, st, detour_surr(p, b, k), gc);
    const bool feasible = a.cacc[2 * B + b] == 0.f;
    float dc;
    if (p.cstr_mode == 1 || (p.cstr_mode == 3 && !feasible)) dc = p.cstr_coef * 2.f * fmaxf(c, 0.f);
    else if (p.cstr_mode == 2) dc = c > 0.f ? p.cstr_coef : 0.f;
    else dc = c <= 0.f ? 1.f / (p.cstr_coef * (c - DETOUR_EPS)) : 0.f;
    const float wgt = dc * p.gpow[k] * p.inv_B;
    lam[0] += wgt * gc[0]; lam[1] += wgt * gc[1]; lam[2] += wgt * gc[2];
  }
#pragma unroll
  for (int j = 0; j < MAXA; ++j)
    if (j < a.act_dim) a.Zb[(size_t)k * a.zs_k + (size_t)b * a.zs_b + j] = abar[j] * g[j];
#pragma unroll
  for (int f = 0; f < NS; ++f) a.lam[(size_t)f * B + b] = lam[f];
}

// single model step (EnvModel.forward inside the wrapper chain, as veh_step_kernel<2> for the plain tracking model):
// next_obs / reward / next_done / next_state of the detour / surrcstr variant; info["constraint"] of the incoming state is
// evaluated by the Python model class (element-wise torch code on the device tensors, like pyth_veh3dofconti_errcstr)
__global__ void veh_step_detour_kernel(const __grid_constant__ KParams p, const float* __restrict__ action,
                                       float* __restrict__ next_obs, float* __restrict__ reward, float* __restrict__ next_done,
                                       float* __restrict__ next_state) {
  const long long gs = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gs >= p.batch) return;
  const int obs_dim = p.pol.obs, P = p.veh_P;
  const VehC vc = veh_const();
  float a[MAXA], s[6];
#pragma unroll
  for (int j = 0; j < MAXA; ++j) {
    float gg = 1.f;
    a[j] = j < 2 ? wrap_action(p, j, action[gs * 2 + j], gg) : 0.f;
  }
#pragma unroll
  for (int f = 0; f < 6; ++f) s[f] = p.state[gs * 6 + f];
  const bool dn = p.done[gs] != 0.f;
  const float* obs = p.obs + gs * obs_dim;
  float* nobs = next_obs + gs * obs_dim;
  RefWindow<2, 1> w;
  w.base = p.reference + gs * (size_t)p.ref_len * 4;
  w.k0 = p.ref_t;
  float q[4];
  w.get(0, q);
  const float ex = s[0] - q[0], ey = s[1] - q[1], ep = angle_normalize(s[2] - q[2]), eu = s[3] - q[3];
  float r = -p.veh_rscale * (p.veh_rc[0] * (ex * ex) + p.veh_rc[1] * (ey * ey) + p.veh_rc[2] * (ep * ep) + p.veh_rc[3] * (eu * eu) +
                             p.veh_rc[4] * (s[5] * s[5]) + p.veh_rc[5] * (a[0] * a[0]) + p.veh_rc[6] * (a[1] * a[1])) +
            p.veh_roff;
  veh_step(vc, s, a);
  w.k0 = p.ref_t + 1;
  float o6[6];
  veh_write_obs<2, 1>(s, w, P, nobs, 1, o6);
  {
    float sn, cs, o4[4];
    sincosf(-s[2], &sn, &cs);
    const float* sp = detour_surr(p, gs, 1);
    ego_obs(s, cs, sn, sp[0], sp[1], sp[2], 0.f, o4);
    nobs[6 + 4 * P] = o4[0]; nobs[6 + 4 * P + 1] = o4[1]; nobs[6 + 4 * P + 2] = o4[2]; nobs[6 + 4 * P + 3] = sp[3];
  }
  w.get(0, q);
  bool md = (fabsf(s[0] - q[0]) > 5.f) || (fabsf(s[1] - q[1]) > p.veh_ydone) ||
            (fabsf(angle_normalize(s[2] - q[2])) > 3.14159265358979323846f);
#pragma unroll
  for (int f = 0; f < 6; ++f) next_state[gs * 6 + f] = s[f];
  if (p.mask_at_done && dn) {     // MaskAtDone: frozen observation, zero reward; info["state"] still advances
    r = 0.f;
    for (int f = 0; f < obs_dim; ++f) nobs[f] = obs[f];
  }
  if (p.mask_at_done) md = md || dn;
  r = shape_reward(p, r);
  reward[gs] = r;
  next_done[gs] = md ? 1.f : 0.f;
}

// [loss | exterior / Lagrangian constraint mean | interior term or #done | #feasible] in fixed order (one block)
__global__ void lw_scalars_detour_kernel(const __grid_constant__ KParams p, const float* __restrict__ vacc,
                                         const float* __restrict__ cacc, const float* __restrict__ dn_last,
                                         float* __restrict__ scalars) {
  __shared__ float s[4][256];
  const long long B = p.batch;
  float l = 0.f, ce = 0.f, third = 0.f, nf = 0.f;
  for (long long i = threadIdx.x; i < B; i += 256) {
    l += -vacc[i] * p.inv_B;
    if (p.cstr_mode != 0) {
      const bool feasible = cacc[2 * B + i] == 0.f;
      const float ca = cacc[i], cb = cacc[B + i];
      if (p.cstr_mode == 3) {
        l += (feasible ? cb / p.cstr_coef : p.cstr_coef * ca) * p.inv_B;
        ce += feasible ? 0.f : ca * p.inv_B;
        third += feasible ? cb / p.cstr_coef * p.inv_B : 0.f;
      } else {
        l += p.cstr_coef * ca * p.inv_B;
        ce += ca * p.inv_B;
      }
      nf += feasible ? 1.f : 0.f;
    }
    if (p.cstr_mode != 3) third += dn_last[i];
  }
  s[0][threadIdx.x] = l; s[1][threadIdx.x] = ce; s[2][threadIdx.x] = third; s[3][threadIdx.x] = nf;
  __syncthreads();
  if (threadIdx.x < 4) {
    float t = 0.f;
    for (int i = 0; i < 256; ++i) t += s[threadIdx.x][i];
    scalars[threadIdx.x] = t;
  }
}

}  // namespace gops
