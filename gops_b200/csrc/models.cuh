// Per-sample environment-model dynamics and their hand-derived adjoints (one thread = one sample).
#pragma once
#include "rollout.cuh"
#include "models_veh.cuh"
#include "models_robot.cuh"

namespace gops {

// ---------------------------------------------------------------------------------------------
// Flags of the wrapper chain.  WrapRt reads them from KParams at run time; WrapFixed<F> fixes them at compile time
// (F: kWrap* bits), so that a kernel built for one chain drops the branches of the others.  A fixed chain with
// kWrapRepeat still reads its repeat count at run time.
// ---------------------------------------------------------------------------------------------
enum : unsigned { kWrapObsScaling = 1, kWrapClipObs = 2, kWrapActionScale = 4, kWrapClipAction = 8, kWrapRepeat = 16 };

__host__ __device__ inline unsigned wrap_bits(const KParams& p) {
  return (p.obs_scaling ? kWrapObsScaling : 0u) | (p.clip_obs ? kWrapClipObs : 0u) |
         (p.action_scale ? kWrapActionScale : 0u) | (p.clip_action ? kWrapClipAction : 0u) |
         (p.repeat_num > 0 ? kWrapRepeat : 0u);
}

struct WrapRt {
  __device__ static __forceinline__ int obs_scaling(const KParams& p) { return p.obs_scaling; }
  __device__ static __forceinline__ int clip_obs(const KParams& p) { return p.clip_obs; }
  __device__ static __forceinline__ int action_scale(const KParams& p) { return p.action_scale; }
  __device__ static __forceinline__ int clip_action(const KParams& p) { return p.clip_action; }
  __device__ static __forceinline__ int repeat_num(const KParams& p) { return p.repeat_num; }
};
template <unsigned F>
struct WrapFixed {
  __device__ static __forceinline__ int obs_scaling(const KParams&) { return (F & kWrapObsScaling) != 0; }
  __device__ static __forceinline__ int clip_obs(const KParams&) { return (F & kWrapClipObs) != 0; }
  __device__ static __forceinline__ int action_scale(const KParams&) { return (F & kWrapActionScale) != 0; }
  __device__ static __forceinline__ int clip_action(const KParams&) { return (F & kWrapClipAction) != 0; }
  __device__ static __forceinline__ int repeat_num(const KParams& p) { return (F & kWrapRepeat) != 0 ? p.repeat_num : 0; }
};

// ---------------------------------------------------------------------------------------------
// Policy output -> model action through tanh squashing + ScaleAction + ClipAction.
//   mlp.py:73-77 / :103-111          a_pol = (hi-lo)/2 * tanh(z) + (hi+lo)/2
//   wrapper/scale_action.py:75-83    clip -> affine -> clip
//   wrapper/clip_action.py:34-40     clip
// a[j]: action handed to the model, g[j] = d a[j] / d z[j] (clip gradient = 1 inside, inclusive).
// ---------------------------------------------------------------------------------------------
// ScaleAction + ClipAction applied to one policy-output component x; gg is multiplied by d(out)/dx
template <class W = WrapRt>
__device__ __forceinline__ float wrap_action(const KParams& p, int j, float x, float& gg) {
  const float lo = p.act_low[j], hi = p.act_high[j];
  if (W::action_scale(p)) {
    const float mn = p.min_action[j], mx = p.max_action[j];
    if (x < mn || x > mx) gg = 0.f;
    x = fminf(fmaxf(x, mn), mx);
    const float q = __fdiv_rn(__fsub_rn(x, mn), __fsub_rn(mx, mn));
    x = __fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), q));
    gg *= __fsub_rn(hi, lo) * __fdiv_rn(1.f, __fsub_rn(mx, mn));
    if (x < lo || x > hi) gg = 0.f;
    x = fminf(fmaxf(x, lo), hi);
  }
  if (W::clip_action(p)) {
    if (x < lo || x > hi) gg = 0.f;
    x = fminf(fmaxf(x, lo), hi);
  }
  return x;
}

// NA: length of the arrays (the kernel's action count, >= na)
template <int NA = MAXA, class W = WrapRt>
__device__ __forceinline__ void process_action(const KParams& p, int na, const float* z, float* a, float* g,
                                               float* apol_out) {
#pragma unroll
  for (int j = 0; j < NA; ++j) {
    if (j >= na) { a[j] = 0.f; g[j] = 0.f; if (apol_out) apol_out[j] = 0.f; continue; }
    const float th = tanhf(z[j]);
    const float x = __fadd_rn(__fmul_rn(p.pol_half[j], th), p.pol_mid[j]);
    float gg = p.pol_half[j] * (1.f - th * th);
    if (apol_out) apol_out[j] = x;
    a[j] = wrap_action<W>(p, j, x, gg);
    g[j] = gg;
  }
}

// ---------------------------------------------------------------------------------------------
// Observation / reward wrappers around the model step (create_env_model.py:104-126), shared by every kernel.
//   wrapper/scale_observation.py    outer obs = (inner obs + shift) * scale
//   wrapper/shaping_reward.py       r = (r + shift) * scale, also for masked (done) samples
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float to_inner(const KParams& p, int f, float x) {
  return p.obs_scaling ? x / p.osc[f] - p.osh[f] : x;
}
__device__ __forceinline__ float to_outer(const KParams& p, int f, float x) {
  return p.obs_scaling ? (x + p.osh[f]) * p.osc[f] : x;
}
__device__ __forceinline__ float shape_reward(const KParams& p, float r) {
  return p.reward_shaping ? (r + p.reward_shift) * p.reward_scale : r;
}
// dL/d(raw reward of step k) of the mean discounted return
__device__ __forceinline__ float reward_adjoint(const KParams& p, int k) {
  return -p.gpow[k] * p.inv_B * (p.reward_shaping ? p.reward_scale : 1.f);
}

// The model step and its adjoint.  A model with constraints (NC > 0) also reads its noise nz and reports / receives the
// constraints of the raw next state (c / cbar); the others take neither.
template <class M>
__device__ __forceinline__ void model_fwd(const KParams& p, float* s, const float* a, const float* nz, float& r, bool& d,
                                          float* c) {
  if constexpr (M::NC > 0) M::step(p, s, a, nz, r, d, c);
  else M::step(p, s, a, r, d);
}
template <class M, bool UNROLL>
__device__ __forceinline__ void model_bwd(const KParams& p, const float* s, const float* a, const float* nz, float rho,
                                          float* lam, float* abar, const float* cbar) {
  if constexpr (M::NC > 0) M::template step_bwd<UNROLL>(p, s, a, nz, rho, lam, abar, cbar);
  else M::template step_bwd<UNROLL>(p, s, a, rho, lam, abar);
}
__host__ __device__ constexpr int nc_slots(int nc) { return nc > 0 ? nc : 1; }
struct NoCstrAdjoint {       // models without constraints: nothing to differentiate
  __device__ void operator()(const float*, float*) const {}
};

// One step of a state==obs model (KIND 0) inside its wrappers, on the outer observation st[0..obs_dim) (in place):
// ScaleObservation -> ActionRepeat (the masked model step repeated with the same action) -> unscale -> ClipObservation.
// When `active` (not frozen by MaskAtDone) r receives the raw reward and dn the new done flag; else both are left alone.
// A model with constraints (no ActionRepeat) steps frozen samples too, as the reference's MaskAtDone does: c receives
// the constraints of that raw step (info["constraint"] is not masked), the frozen observation stays.
template <class M, class W = WrapRt>
__device__ __forceinline__ void wrapped_step(const KParams& p, int obs_dim, float* st, const float* a, bool active,
                                             float& r, bool& dn, const float* nz = nullptr, float* c = nullptr) {
  constexpr int NS = M::NS;
  float in[NS];
#pragma unroll
  for (int f = 0; f < NS; ++f) in[f] = (W::obs_scaling(p) && f < obs_dim) ? st[f] / p.osc[f] - p.osh[f] : st[f];
  if constexpr (M::NC > 0) {
    float nx[NS], rj;
    bool md;
#pragma unroll
    for (int f = 0; f < NS; ++f) nx[f] = in[f];
    model_fwd<M>(p, nx, a, nz, rj, md, c);
    if (active) {
#pragma unroll
      for (int f = 0; f < NS; ++f) in[f] = nx[f];
      r = rj;
      dn = md;
    }
  } else if (active) {
    bool md = false;
    const int reps = W::repeat_num(p) > 0 ? W::repeat_num(p) : 1;
    float rsum = 0.f, rj = 0.f;
    for (int j = 0; j < reps; ++j) {
      M::step(p, in, a, rj, md);
      rsum += rj;
    }
    r = (W::repeat_num(p) > 0 && p.sum_reward) ? rsum : rj;
    dn = md;
  }
#pragma unroll
  for (int f = 0; f < NS; ++f) {
    float o = (W::obs_scaling(p) && f < obs_dim) ? (in[f] + p.osh[f]) * p.osc[f] : in[f];
    if (W::clip_obs(p)) o = fminf(fmaxf(o, p.obs_low[f]), p.obs_high[f]);
    st[f] = o;
  }
}

// Adjoint of wrapped_step: st = outer observation before the step, lam = adjoint of the outer observation after it
// (in) / before it (out), rho = dL/d(raw reward), abar[j] += dL/d a[j].  Chain of the step:
//   obs_k -(1/scale, -shift)-> inner_0 -[model step x reps, same action]-> inner_reps -(+shift, *scale)-> clip -> obs_k+1
// NA: length of abar (the kernel's action count; M reads a[0, NA) and writes at most MAXA adjoints).  UNROLL: passed to
// M::step_bwd.  Models with constraints: cbar_of(c, cbar) turns the constraints of the raw step into their adjoints; a
// frozen sample (!active) passes lam through unchanged and adds only what the constraints pull back.
template <class M, int NA = MAXA, class W = WrapRt, bool UNROLL = false, class CB = NoCstrAdjoint>
__device__ __forceinline__ void wrapped_step_bwd(const KParams& p, int obs_dim, const float* st, const float* a,
                                                 float rho, float* lam, float* abar, const float* nz = nullptr,
                                                 bool active = true, CB cbar_of = CB()) {
  constexpr int NS = M::NS;
  const int reps = W::repeat_num(p) > 0 ? W::repeat_num(p) : 1;
  float in0[NS], cur[NS], c[nc_slots(M::NC)], cbar[nc_slots(M::NC)], keep[NS];
#pragma unroll
  for (int f = 0; f < NS; ++f) in0[f] = (W::obs_scaling(p) && f < obs_dim) ? st[f] / p.osc[f] - p.osh[f] : st[f];
  if constexpr (M::NC > 0) {
    if (!active) {            // obs_k+1 = clip(obs_k): the adjoint passes where obs_k is inside the bounds
#pragma unroll
      for (int f = 0; f < NS; ++f) {
        keep[f] = (W::clip_obs(p) && (st[f] < p.obs_low[f] || st[f] > p.obs_high[f])) ? 0.f : lam[f];
        lam[f] = 0.f;
      }
      rho = 0.f;
    }
  }
  if (W::clip_obs(p) || M::NC > 0) {   // the raw next state: clip passes gradient only where it is inside; constraints
    float rr;
    bool md;
#pragma unroll
    for (int f = 0; f < NS; ++f) cur[f] = in0[f];
    for (int j = 0; j < reps; ++j) model_fwd<M>(p, cur, a, nz, rr, md, c);
    if constexpr (M::NC > 0) cbar_of(c, cbar);
    if (W::clip_obs(p)) {
#pragma unroll
      for (int f = 0; f < NS; ++f) {
        const float o = (W::obs_scaling(p) && f < obs_dim) ? (cur[f] + p.osh[f]) * p.osc[f] : cur[f];
        if (o < p.obs_low[f] || o > p.obs_high[f]) lam[f] = 0.f;
      }
    }
  }
  if (W::obs_scaling(p)) {
#pragma unroll
    for (int f = 0; f < NS; ++f)
      if (f < obs_dim) lam[f] *= p.osc[f];
  }
  for (int j = reps - 1; j >= 0; --j) {
    float rr, aj[MAXA];
    bool md;
#pragma unroll
    for (int f = 0; f < NS; ++f) cur[f] = in0[f];
    for (int q = 0; q < j; ++q) model_fwd<M>(p, cur, a, nz, rr, md, c);      // state before repeat j
    const float rho_j = (W::repeat_num(p) == 0 || p.sum_reward || j == reps - 1) ? rho : 0.f;
#pragma unroll
    for (int q = 0; q < MAXA; ++q) aj[q] = 0.f;
    model_bwd<M, UNROLL>(p, cur, a, nz, rho_j, lam, aj, cbar);
#pragma unroll
    for (int q = 0; q < NA; ++q) abar[q] += aj[q];
  }
  if (W::obs_scaling(p)) {
#pragma unroll
    for (int f = 0; f < NS; ++f)
      if (f < obs_dim) lam[f] /= p.osc[f];
  }
  if constexpr (M::NC > 0) {
    if (!active) {
#pragma unroll
      for (int f = 0; f < NS; ++f) lam[f] += keep[f];
    }
  }
}

// =============================================================================================
// pyth_idpendulum   (env_ocp/env_model/pyth_idpendulum_model.py)
// state s = [p, th1, th2, pdot, th1dot, th2dot]; 5 explicit-Euler sub-steps of tau = dt/5 with
// acceleration x = M(th)^-1 f(th, thdot, u), u = 500 a.
// =============================================================================================
struct IdpC {
  float A, Bc, Cc, D, E, F, G1, G2, tau;
};
__device__ __forceinline__ IdpC idp_const() {
  // constants are formed in double exactly as the python expressions (:21-29, :52-90), then cast
  constexpr double m = 9.42477796, m1 = 4.1033127, m2 = 4.1033127, l1 = 0.6, l2 = 0.6, g = 9.81;
  IdpC c;
  c.A = (float)(m + m1 + m2);
  c.Bc = (float)(l1 * (0.5 * m1 + m2));
  c.Cc = (float)(0.5 * m2 * l2);
  c.D = (float)(l1 * l1 * (0.3333 * m1 + m2));
  c.E = (float)(0.5 * l1 * l2 * m2);
  c.F = (float)(0.3333 * l2 * l2 * m2);
  c.G1 = (float)(g * (0.5 * m1 + m2) * l1);
  c.G2 = (float)(g * 0.5 * l2 * m2);
  c.tau = (float)(0.01 / 5);
  return c;
}

struct IdpAux {
  float s1, c1, s2, c2, s12, c12;
  float i00, i01, i02, i11, i12, i22;  // symmetric inverse mass matrix
  float x0, x1, x2;                    // accelerations
};
// what the adjoint keeps of a sub-step's idp_eval: the MUFU sines / cosines and the IEEE reciprocal of det M
struct IdpKeep {
  float s1, c1, s2, c2, s12, c12, r;
};

// q from the sines / cosines in k and the angular velocities v1, v2.  FWD: forms k.r = 1 / det M, else takes it from k
// (the same value: the mass matrix depends on the cosines alone)
template <bool FWD>
__device__ __forceinline__ void idp_eval_k(float v1, float v2, float u, const IdpC& c, IdpKeep& k, IdpAux& q) {
  q.s1 = k.s1; q.c1 = k.c1; q.s2 = k.s2; q.c2 = k.c2; q.s12 = k.s12; q.c12 = k.c12;
  const float a = c.A, b = c.Bc * q.c1, cc = c.Cc * q.c2, d = c.D, e = c.E * q.c12, f = c.F;
  const float f0 = (c.Bc * (v1 * v1)) * q.s1 + (c.Cc * (v2 * v2)) * q.s2 + u;
  const float f1 = (-c.E * (v2 * v2)) * q.s12 + c.G1 * q.s1;
  // rounded as written (as the compiler contracted it before q was kept): its choice depends on the other uses of q
  const float f2 = __fmaf_rn(c.G2, q.s2, __fmul_rn(c.E * (v1 * v1), q.s12));
  const float C00 = d * f - e * e, C01 = cc * e - b * f, C02 = b * e - cc * d;
  const float C11 = a * f - cc * cc, C12 = b * cc - a * e, C22 = a * d - b * b;
  if constexpr (FWD) {
    const float det = a * C00 + b * C01 + cc * C02;
    k.r = 1.f / det;
  }
  const float r = k.r;
  q.i00 = C00 * r; q.i01 = C01 * r; q.i02 = C02 * r; q.i11 = C11 * r; q.i12 = C12 * r; q.i22 = C22 * r;
  q.x0 = q.i00 * f0 + q.i01 * f1 + q.i02 * f2;
  q.x1 = q.i01 * f0 + q.i11 * f1 + q.i12 * f2;
  q.x2 = q.i02 * f0 + q.i12 * f1 + q.i22 * f2;
}

// one sub-step in place; k receives what the adjoint keeps of it (IdpKeep)
__device__ __forceinline__ void idp_substep(float* s, float u, const IdpC& c, IdpKeep& k) {
  // pendulum angles stay within a few radians: the MUFU sine/cosine (abs. error ~5e-7 on [-pi, pi]) is inside
  // the fp32 noise of the reference here; the parity tests (loss 1e-4, gradient 2e-4, exact termination step) gate it
  __sincosf(s[1], &k.s1, &k.c1);
  __sincosf(s[2], &k.s2, &k.c2);
  __sincosf(s[1] - s[2], &k.s12, &k.c12);
  IdpAux q;
  idp_eval_k<true>(s[4], s[5], u, c, k, q);
  const float t = c.tau;
  const float n0 = s[0] + t * s[3], n1 = s[1] + t * s[4], n2 = s[2] + t * s[5];
  s[3] += t * q.x0; s[4] += t * q.x1; s[5] += t * q.x2;
  s[0] = n0; s[1] = n1; s[2] = n2;
}

// adjoint of one sub-step: lam (adjoint of s_next) -> lam (adjoint of s); ubar += dL/du.  v1, v2: s[4], s[5];
// q: idp_eval of (s, u), the only other use of s
__device__ __forceinline__ void idp_substep_bwd(float v1, float v2, const IdpAux& q, const IdpC& c, float* lam,
                                                float& ubar) {
  const float t = c.tau;
  const float xb0 = t * lam[3], xb1 = t * lam[4], xb2 = t * lam[5];
  // w = M^-T xb (M symmetric) is the adjoint of f; the adjoint of M is -w x^T.  w2 and m02 are rounded as written (as
  // the compiler contracted them when q was formed in this function): its choice depends on where q comes from
  const float w0 = q.i00 * xb0 + q.i01 * xb1 + q.i02 * xb2;
  const float w1 = q.i01 * xb0 + q.i11 * xb1 + q.i12 * xb2;
  const float w2 = __fmaf_rn(q.i22, xb2, __fmaf_rn(q.i02, xb0, __fmul_rn(q.i12, xb1)));
  const float m01 = -(w0 * q.x1 + w1 * q.x0), m02 = -__fmaf_rn(w0, q.x2, __fmul_rn(w2, q.x0));
  const float m12 = -(w1 * q.x2 + w2 * q.x1);
  float th1b = m01 * (-c.Bc * q.s1) + m12 * (-c.E * q.s12);
  float th2b = m02 * (-c.Cc * q.s2) + m12 * (c.E * q.s12);
  // f0 = Bc v1^2 s1 + Cc v2^2 s2 + u
  th1b += w0 * (c.Bc * v1 * v1 * q.c1);
  th2b += w0 * (c.Cc * v2 * v2 * q.c2);
  float v1b = w0 * (2.f * c.Bc * v1 * q.s1);
  float v2b = w0 * (2.f * c.Cc * v2 * q.s2);
  ubar += w0;
  // f1 = -E v2^2 s12 + G1 s1
  th1b += w1 * (-c.E * v2 * v2 * q.c12 + c.G1 * q.c1);
  th2b += w1 * (c.E * v2 * v2 * q.c12);
  v2b += w1 * (-2.f * c.E * v2 * q.s12);
  // f2 = E v1^2 s12 + G2 s2
  th1b += w2 * (c.E * v1 * v1 * q.c12);
  th2b += w2 * (-c.E * v1 * v1 * q.c12 + c.G2 * q.c2);
  v1b += w2 * (2.f * c.E * v1 * q.s12);
  const float l0 = lam[0], l1 = lam[1], l2 = lam[2];
  lam[1] = l1 + th1b;
  lam[2] = l2 + th2b;
  lam[3] = lam[3] + t * l0;
  lam[4] = lam[4] + t * l1 + v1b;
  lam[5] = lam[5] + t * l2 + v2b;
}

struct ModelIdp {
  static constexpr int NS = 6, KIND = 0, NC = 0;
  // forward: s <- next state; returns raw model reward and done   (:199-216, :126-172)
  __device__ static __forceinline__ void step(const KParams&, float* s, const float* a, float& rew, bool& done) {
    const IdpC c = idp_const();
    const float u = 500.f * a[0];
    IdpKeep k;
#pragma unroll 1
    for (int j = 0; j < 5; ++j) idp_substep(s, u, c, k);
    const float dist = 0.f * (s[0] * s[0]) + 5.f * (s[1] * s[1]) + 10.f * (s[2] * s[2]);
    const float vel = 0.5f * (s[3] * s[3]) + 0.5f * (s[4] * s[4]) + 1.f * (s[5] * s[5]);
    rew = 10.f - dist - vel - a[0] * a[0];
    const float tip_y = 0.6f * cosf(s[1]) + 0.6f * cosf(s[2]);
    done = (tip_y <= 1.0f) || (fabsf(s[0]) >= 15.f);
  }
  // backward: s = state BEFORE the step, lam = adjoint of the next state (in) / of s (out),
  // rho = dL/d(raw reward of this step).  abar[j] = dL/d a[j].  UNROLL: the sub-step loops unrolled, so that what the
  // adjoint keeps of each sub-step (45 floats in all) stays in registers; else they are rolled over thread-local arrays.
  template <bool UNROLL = false>
  __device__ static __forceinline__ void step_bwd(const KParams&, const float* s, const float* a, float rho, float* lam,
                                                  float* abar) {
    const IdpC c = idp_const();
    const float u = 500.f * a[0];
    // what the adjoint of sub-step j needs of its state: the angular velocities and IdpKeep, formed once here
    float vj[5][2], s5[6];
    IdpKeep kj[5];
#pragma unroll
    for (int f = 0; f < 6; ++f) s5[f] = s[f];
#pragma unroll (UNROLL ? 5 : 1)
    for (int j = 0; j < 5; ++j) {
      vj[j][0] = s5[4];
      vj[j][1] = s5[5];
      idp_substep(s5, u, c, kj[j]);
    }
    // reward is evaluated on the post-step state
    lam[1] += rho * (-10.f * s5[1]);
    lam[2] += rho * (-20.f * s5[2]);
    lam[3] += rho * (-s5[3]);
    lam[4] += rho * (-s5[4]);
    lam[5] += rho * (-2.f * s5[5]);
    float ubar = 0.f;
#pragma unroll (UNROLL ? 5 : 1)
    for (int j = 4; j >= 0; --j) {
      IdpAux q;
      idp_eval_k<false>(vj[j][0], vj[j][1], u, c, kj[j], q);
      idp_substep_bwd(vj[j][0], vj[j][1], q, c, lam, ubar);
    }
    abar[0] = rho * (-2.f * a[0]) + 500.f * ubar;
  }
};

// =============================================================================================
// pyth_lq   (env_ocp/resources/lq_base.py:89-141, :343-354)   zero-padded to LQN x MAXA
// =============================================================================================
struct ModelLq {
  static constexpr int NS = LQN, KIND = 0, NC = 0;
  __device__ static __forceinline__ void step(const KParams& p, float* s, const float* a, float& rew, bool& done) {
    float rs = 0.f, ra = 0.f, tmp[LQN];
#pragma unroll
    for (int i = 0; i < LQN; ++i) rs += (s[i] * s[i]) * p.lq_Q[i];
#pragma unroll
    for (int j = 0; j < MAXA; ++j) ra += (a[j] * a[j]) * p.lq_R[j];
    rew = p.lq_rs * (p.lq_rsh - 1.0f * (rs + ra));
#pragma unroll
    for (int i = 0; i < LQN; ++i) {
      float bu = 0.f;
#pragma unroll
      for (int j = 0; j < MAXA; ++j) bu = fmaf(p.lq_B[i * MAXA + j], a[j], bu);
      tmp[i] = bu * p.lq_dt + s[i];
    }
#pragma unroll
    for (int i = 0; i < LQN; ++i) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < LQN; ++j) acc = fmaf(p.lq_inv_IA[i * LQN + j], tmp[j], acc);
      s[i] = acc;
    }
    done = false;
  }
  template <bool = false>
  __device__ static __forceinline__ void step_bwd(const KParams& p, const float* s, const float* a, float rho,
                                                  float* lam, float* abar) {
    float tb[LQN];
#pragma unroll
    for (int j = 0; j < LQN; ++j) {
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < LQN; ++i) acc = fmaf(p.lq_inv_IA[i * LQN + j], lam[i], acc);
      tb[j] = acc;
    }
    const float rr = rho * p.lq_rs;
#pragma unroll
    for (int j = 0; j < MAXA; ++j) {
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < LQN; ++i) acc = fmaf(p.lq_B[i * MAXA + j], tb[i], acc);
      abar[j] = p.lq_dt * acc + rr * (-2.f * p.lq_R[j] * a[j]);
    }
#pragma unroll
    for (int i = 0; i < LQN; ++i) lam[i] = tb[i] + rr * (-2.f * p.lq_Q[i] * s[i]);
  }
};

// =============================================================================================
// Vehicle models: the observation is a function of (robot state, reference window); the kernel keeps the
// robot state (+ reference time for pyth_veh3dofconti) per thread and rebuilds observations on the fly.
// KIND 1: pyth_veh3dofconti (analytic reference generator, window kept in a per-CTA global scratch)
// KIND 2: env_gen_ocp veh3dof_tracking (window = slice of the caller's reference tensor)
// =============================================================================================
struct ModelVehConti {
  static constexpr int NS = 7, KIND = 1, NC = 2;   // x, y, phi, u, v, w, ref_time; NC: (|y_err|, |u_err|) constraints
  // reward from the INCOMING inner observation o (Veh3dofcontiModel.compute_reward :161-177)
  __device__ static __forceinline__ float reward(const float* o, const float* a) {
    return -(0.04f * (o[0] * o[0]) + 0.04f * (o[1] * o[1]) + 0.02f * (o[2] * o[2]) + 0.02f * (o[3] * o[3]) +
             0.01f * (o[5] * o[5]) + 0.01f * (a[0] * a[0]) + 0.01f * (a[1] * a[1]));
  }
  // termination test on the NEW inner observation o
  __device__ static __forceinline__ bool done(const float* o) {
    return (fabsf(o[0]) > 10.f) || (fabsf(o[1]) > 10.f) || (fabsf(o[2]) > 3.14159265358979323846f);
  }
  // adjoint of reward(): ob[0..5] = dL/d o (entry 4 untouched), abar += dL/d a; rho = dL/d(reward)
  __device__ static __forceinline__ void reward_bwd(const float* o, const float* a, float rho, float* ob, float* abar) {
    abar[0] += rho * (-0.02f * a[0]);
    abar[1] += rho * (-0.02f * a[1]);
    ob[0] = rho * (-0.08f * o[0]); ob[1] = rho * (-0.08f * o[1]);
    ob[2] = rho * (-0.04f * o[2]); ob[3] = rho * (-0.04f * o[3]);
    ob[5] = rho * (-0.02f * o[5]);
  }
};
struct ModelVehTrack {
  static constexpr int NS = 6, KIND = 2, NC = 0;
  // reward from the CURRENT state s against reference point q = reference[:, t] (veh3dof_tracking_model.py:59-73)
  __device__ static __forceinline__ float reward(const float* s, const float* q, const float* a) {
    const float ex = s[0] - q[0], ey = s[1] - q[1], ep = angle_normalize(s[2] - q[2]), eu = s[3] - q[3];
    return -(0.04f * (ex * ex) + 0.04f * (ey * ey) + 0.02f * (ep * ep) + 0.02f * (eu * eu) + 0.01f * (s[5] * s[5]) +
             0.01f * (a[0] * a[0]) + 0.01f * (a[1] * a[1]));
  }
  // termination test of the new state s against reference[:, t + 1]
  __device__ static __forceinline__ bool done(const float* s, const float* q) {
    return (fabsf(s[0] - q[0]) > 5.f) || (fabsf(s[1] - q[1]) > 2.f) ||
           (fabsf(angle_normalize(s[2] - q[2])) > 3.14159265358979323846f);
  }
  // adjoint of reward(): lam += dL/d s, abar += dL/d a; rho = dL/d(reward)
  __device__ static __forceinline__ void reward_bwd(const float* s, const float* q, const float* a, float rho, float* lam,
                                                    float* abar) {
    abar[0] += rho * (-0.02f * a[0]);
    abar[1] += rho * (-0.02f * a[1]);
    lam[0] += rho * (-0.08f * (s[0] - q[0]));
    lam[1] += rho * (-0.08f * (s[1] - q[1]));
    lam[2] += rho * (-0.04f * angle_normalize(s[2] - q[2]));
    lam[3] += rho * (-0.04f * (s[3] - q[3]));
    lam[5] += rho * (-0.02f * s[5]);
  }
};

// Accessor of the (P+1)-point reference window of one sample at horizon step k.
template <int KIND, int NT>
struct RefWindow {
  const float* base;   // KIND 1: ext_ref + tid (point-major, stride NT)   KIND 2: reference + gs*L*4
  int k0;              // first point of the window
  __device__ __forceinline__ void get(int i, float* q) const {
    if (KIND == 1) {
      const float* b = base + (size_t)(k0 + i) * 4 * NT;
      q[0] = b[0]; q[1] = b[NT]; q[2] = b[2 * NT]; q[3] = b[3 * NT];
    } else {
      const float4 v = *reinterpret_cast<const float4*>(base + (size_t)(k0 + i) * 4);
      q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
    }
  }
};

// obs = get_obs(state, window) written into column `col` of X (row stride ld); returns first 6 entries in o6
template <int KIND, int NT>
__device__ __forceinline__ void veh_write_obs(const float* s, const RefWindow<KIND, NT>& w, int P, float* col, int ld,
                                              float* o6) {
  float sn, cs;
  sincosf(-s[2], &sn, &cs);
  float q[4], o4[4];
  w.get(0, q);
  ego_obs(s, cs, sn, q[0], q[1], q[2], q[3], o4);
  o6[0] = o4[0]; o6[1] = o4[1]; o6[2] = o4[2]; o6[3] = o4[3]; o6[4] = s[4]; o6[5] = s[5];
#pragma unroll
  for (int f = 0; f < 6; ++f) col[f * ld] = o6[f];
  for (int i = 1; i <= P; ++i) {
    w.get(i, q);
    ego_obs(s, cs, sn, q[0], q[1], q[2], q[3], o4);
    float* c = col + (6 + 4 * (i - 1)) * ld;
    c[0] = o4[0]; c[ld] = o4[1]; c[2 * ld] = o4[2]; c[3 * ld] = o4[3];
  }
}

// ScaleObservationModel on a freshly written observation column: obs <- (obs + shift) * scale
__device__ __forceinline__ void veh_scale_obs(const KParams& p, int obs_dim, float* col, int ld) {
  for (int f = 0; f < obs_dim; ++f) col[f * ld] = (col[f * ld] + p.osh[f]) * p.osc[f];
}

// adjoint of get_obs w.r.t. the robot state: lam[0..5] += O^T xbar, xbar read from column `col` of X;
// extra6 = additional adjoint on the first 6 observation entries (reward-on-observation term)
template <int KIND, int NT>
__device__ __forceinline__ void veh_obs_bwd(const float* s, const RefWindow<KIND, NT>& w, int P, const float* col,
                                            int ld, const float* extra6, const float* osc, float* lam) {
  float sn, cs;
  sincosf(-s[2], &sn, &cs);
  float bx = 0.f, by = 0.f, bphi = 0.f, bu = 0.f;
  for (int i = 0; i <= P; ++i) {
    float q[4];
    w.get(i, q);
    const int f0 = i == 0 ? 0 : (6 + 4 * (i - 1));
    const float* c = col + f0 * ld;
    float ox = c[0], oy = c[ld], op = c[2 * ld], ou = c[3 * ld];
    if (osc != nullptr) { ox *= osc[f0]; oy *= osc[f0 + 1]; op *= osc[f0 + 2]; ou *= osc[f0 + 3]; }   // outer -> inner
    if (i == 0) { ox += extra6[0]; oy += extra6[1]; op += extra6[2]; ou += extra6[3]; }
    const float dx = q[0] - s[0], dy = q[1] - s[1];
    const float vx = dx * cs - dy * sn, vy = dx * sn + dy * cs;   // the forward observation entries
    bx += -cs * ox - sn * oy;
    by += sn * ox - cs * oy;
    bphi += vy * ox - vx * oy - op;      // d cos(-phi)/dphi = sin(-phi), d sin(-phi)/dphi = -cos(-phi)
    bu += -ou;
  }
  lam[0] += bx; lam[1] += by; lam[2] += bphi; lam[3] += bu;
  lam[4] += col[4 * ld] * (osc != nullptr ? osc[4] : 1.f) + extra6[4];
  lam[5] += col[5 * ld] * (osc != nullptr ? osc[5] : 1.f) + extra6[5];
}

}  // namespace gops
