// pyth_mobilerobot (env_ocp/env_model/pyth_mobilerobot_model.py): an ego robot tracking the path y = 0 past one moving
// obstacle, state == observation (13 entries), one obstacle-distance constraint, obstacle noise read from a buffer.
#pragma once
#include "rollout.cuh"

namespace gops {

// ClipObservation bounds of the model (pyth_mobilerobot_model.py:36-45), fp32 of the python values
constexpr double kRobotPi = 3.14159265358979323846;
constexpr float kRobotObsLow[13] = {-30.f, -30.f, (float)(-2 * kRobotPi), -1.f, (float)(-kRobotPi / 2), -30.f,
                                    (float)(-kRobotPi), -2.f, -30.f, -30.f, (float)(-2 * kRobotPi), -1.f,
                                    (float)(-kRobotPi / 2)};
constexpr float kRobotObsHigh[13] = {60.f, 30.f, (float)(2 * kRobotPi), 1.f, (float)(kRobotPi / 2), 30.f,
                                     (float)kRobotPi, 2.f, 30.f, 30.f, (float)(2 * kRobotPi), 1.f, (float)(kRobotPi / 2)};

// state s = [x, y, theta, v, w | e_y, e_theta, e_v | obstacle x, y, theta, v, w]; action a = commanded (v, w) of the ego.
// Robot.f_xu (:136-178), dt = 0.2: rate-limited commands, then a unicycle step.  The obstacle is its own command (so its
// rate limit is clamp(0)) plus noise 0.5 n, n = float32(normal(0, (0.03, 0.02))) per sample, read from nz[0..1]; the ego's
// draws have std 0.  The constraint is 0.89 - |p_obstacle - p_ego| of the RAW next state (radius 0.37 twice + margin
// 0.15).  The forward arithmetic is rounded as torch evaluates it (explicit _rn: no contraction), so that done flags and
// safe flags sit where the reference puts them.
struct ModelMobileRobot {
  static constexpr int NS = 13, KIND = 0, NC = 1, NZ = 2;   // NZ: noise draws per sample and step
  struct Lim {
    float dv, dw, vmax, wmax, T;
  };
  __device__ static __forceinline__ Lim lim() {
    // python doubles -v_delta_max * T etc., cast by torch.clamp to the tensor's fp32
    return {(float)(1.8 * 0.2), (float)(0.8 * 0.2), 0.4f, (float)(kRobotPi / 2), 0.2f};
  }
  __device__ static __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
  // one unicycle of f_xu on s[0..4] with commands (vc, wc) already formed
  __device__ static __forceinline__ void unicycle(float* s, float vc, float wc, float T, float c, float sn) {
    s[0] = __fadd_rn(s[0], __fmul_rn(__fmul_rn(T, c), vc));
    s[1] = __fadd_rn(s[1], __fmul_rn(__fmul_rn(T, sn), vc));
    s[2] = __fadd_rn(s[2], __fmul_rn(T, wc));
    s[3] = vc;
    s[4] = wc;
  }
  __device__ static __forceinline__ float constraint(const float* s) {
    const float dx = __fsub_rn(s[8], s[0]), dy = __fsub_rn(s[9], s[1]);
    return __fsub_rn((float)(0.74 / 2 + 0.74 / 2 + 0.15), sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))));
  }
  // forward: s <- raw next state; rew, done; c[0] = constraint of the raw next state
  __device__ static __forceinline__ void step(const KParams&, float* s, const float* a, const float* nz, float& rew,
                                              bool& done, float* c) {
    const Lim L = lim();
    const float vc = clampf(__fadd_rn(s[3], clampf(__fsub_rn(a[0], s[3]), -L.dv, L.dv)), -L.vmax, L.vmax);
    const float wc = clampf(__fadd_rn(s[4], clampf(__fsub_rn(a[1], s[4]), -L.dw, L.dw)), -L.wmax, L.wmax);
    const float ov = __fadd_rn(clampf(s[11], -L.vmax, L.vmax), __fmul_rn(nz[0], 0.5f));
    const float ow = __fadd_rn(clampf(s[12], -L.wmax, L.wmax), __fmul_rn(nz[1], 0.5f));
    float c0, s0, c1, s1;
    sincosf(s[2], &s0, &c0);
    sincosf(s[10], &s1, &c1);
    unicycle(s, vc, wc, L.T, c0, s0);
    unicycle(s + 8, ov, ow, L.T, c1, s1);
    s[5] = s[1];                        // tracking error against y = 0, phi = 0
    s[6] = s[2];
    s[7] = __fsub_rn(s[3], 0.3f);
    const float ey = s[5], et = s[6], ev = s[7];
    const float rt = __fsub_rn(__fsub_rn(__fmul_rn(-1.4f, __fmul_rn(ey, ey)), __fmul_rn(et, et)), __fmul_rn(16.f, __fmul_rn(ev, ev)));
    const float ra = __fsub_rn(__fmul_rn(-0.2f, __fmul_rn(a[0], a[0])), __fmul_rn(0.5f, __fmul_rn(a[1], a[1])));
    rew = __fadd_rn(rt, ra);
    c[0] = constraint(s);
    done = s[0] < -2.f || fabsf(s[1]) > 4.f || c[0] > 0.15f;
  }
  // backward: s = state BEFORE the step, lam = adjoint of the raw next state (in) / of s (out), rho = dL/d(reward),
  // cbar[0] = dL/d(constraint); abar[j] += dL/d a[j].  torch.clamp passes the gradient on the closed interval.
  template <bool = false>
  __device__ static __forceinline__ void step_bwd(const KParams&, const float* s, const float* a, const float* nz,
                                                  float rho, float* lam, float* abar, const float* cbar) {
    const Lim L = lim();
    auto inside = [](float x, float lo, float hi) { return (x >= lo && x <= hi) ? 1.f : 0.f; };
    const float dv = __fsub_rn(a[0], s[3]), dw = __fsub_rn(a[1], s[4]);
    const float gdv = inside(dv, -L.dv, L.dv), gdw = inside(dw, -L.dw, L.dw);
    const float uv = __fadd_rn(s[3], clampf(dv, -L.dv, L.dv)), uw = __fadd_rn(s[4], clampf(dw, -L.dw, L.dw));
    const float guv = inside(uv, -L.vmax, L.vmax), guw = inside(uw, -L.wmax, L.wmax);
    const float vc = clampf(uv, -L.vmax, L.vmax), wc = clampf(uw, -L.wmax, L.wmax);
    const float gov = inside(s[11], -L.vmax, L.vmax), gow = inside(s[12], -L.wmax, L.wmax);
    const float ov = __fadd_rn(clampf(s[11], -L.vmax, L.vmax), __fmul_rn(nz[0], 0.5f));
    float c0, s0, c1, s1;
    sincosf(s[2], &s0, &c0);
    sincosf(s[10], &s1, &c1);
    float n[NS];
#pragma unroll
    for (int f = 0; f < NS; ++f) n[f] = s[f];
    unicycle(n, vc, wc, L.T, c0, s0);
    unicycle(n + 8, ov, __fadd_rn(clampf(s[12], -L.wmax, L.wmax), __fmul_rn(nz[1], 0.5f)), L.T, c1, s1);
    const float ey = n[1], et = n[2], ev = __fsub_rn(n[3], 0.3f);
    // constraint: c = 0.89 - sqrt(dx^2 + dy^2), dx = ox' - x', dy = oy' - y'
    const float dx = n[8] - n[0], dy = n[9] - n[1];
    const float rinv = 1.f / sqrtf(dx * dx + dy * dy);
    const float cx = cbar[0] * dx * rinv, cy = cbar[0] * dy * rinv;   // dL/d(x', y'); the obstacle gets the negatives
    // adjoints of the raw next state, with the tracking-error entries and the reward folded in
    const float gx = lam[0] + cx;
    const float gy = lam[1] + lam[5] + rho * (-2.8f * ey) + cy;
    const float gt = lam[2] + lam[6] + rho * (-2.f * et);
    const float gvc = lam[3] + lam[7] + rho * (-32.f * ev) + gx * (L.T * c0) + gy * (L.T * s0);
    const float gwc = lam[4] + gt * L.T;
    const float gox = lam[8] - cx, goy = lam[9] - cy, got = lam[10];
    const float gov_ = lam[11] + gox * (L.T * c1) + goy * (L.T * s1);
    const float gow_ = lam[12] + got * L.T;
    lam[0] = gx;
    lam[1] = gy;
    lam[2] = gt + gx * (L.T * -s0 * vc) + gy * (L.T * c0 * vc);
    lam[3] = gvc * guv * (1.f - gdv);
    lam[4] = gwc * guw * (1.f - gdw);
    lam[5] = lam[6] = lam[7] = 0.f;
    lam[8] = gox;
    lam[9] = goy;
    lam[10] = got + gox * (L.T * -s1 * ov) + goy * (L.T * c1 * ov);
    lam[11] = gov_ * gov;
    lam[12] = gow_ * gow;
    abar[0] += gvc * guv * gdv + rho * (-0.4f * a[0]);
    abar[1] += gwc * guw * gdw + rho * (-1.0f * a[1]);
  }
};

}  // namespace gops
