// The fused rollout kernel template: forward sweep, terminal value, reverse sweep, gradient partials.
#pragma once
#include "models.cuh"
#include "mlp_tc_full.cuh"

namespace gops {

// SPIL's constraint-to-cost transform (spil.py:224-232): Phi(c) = (1 + tau m1) / (1 + m2 tau exp(clamp(c / tau, -10, 5)))
// with m1 = 1, m2 = 0.45, tau = 0.07, constants formed in python doubles and applied to fp32 tensors.  dlog = d log Phi / dc
// = -m2 e / (1 + m2 tau e) inside the clamp range, bounds included (torch's clamp passes the gradient there), else 0.
__device__ __forceinline__ float spil_phi(float c, float& dlog) {
  const float y = c / (float)0.07;
  const float e = expf(fminf(fmaxf(y, -10.f), 5.f));
  const float den = 1.f + (float)(0.45 * 0.07) * e;
  dlog = (y >= -10.f && y <= 5.f) ? -0.45f * e / den : 0.f;
  return (float)(1.0 + 0.07) / den;
}

// SPIL's per-sample constraint record of one step, constraints c[0, NC) (NC <= 2): the value pass keeps one safe-so-far
// flag per constraint (traj_issafe *= constraint <= 0, spil.py:200, 207), the policy pass the running product of
// Phi(constraint) (c_mul = c_mul * Phi(c), spil.py:240-252)
template <int NC>
__device__ __forceinline__ void spil_track(bool pev, const float* c, float& ca, float& cb) {
  if (pev) {
    ca = c[0] <= 0.f ? ca : 0.f;
    if (NC > 1) cb = c[1] <= 0.f ? cb : 0.f;
  } else {
    float dl;
    ca *= spil_phi(c[0], dl);
    if (NC > 1) cb *= spil_phi(c[1], dl);
  }
}

// One CTA = NT threads = NT samples per chunk; MLP GEMMs run over SUB = NT/S sub-tiles of S samples that
// reuse one set of activation tiles; the per-sample dynamics (forward and adjoint) run on every thread.
// HD = 64: weights (TMA-staged), weight-gradient accumulators and X live in shared memory.
// HD = 256 (WG): they do not fit (519 KB of weights) -> weights are read from the packed blob in global memory
// (L2 resident, generic loads), gradients accumulate directly in this CTA's global partial, X is a per-CTA global
// scratch; only the activation tiles stay in shared memory.
// (The wgmma rollout kernel is rollout_tc2.cuh; this template is the mma.sync / FFMA family.)
template <class M, int HD, int S, int NT, int ALG>
__global__ void __launch_bounds__(NT, 1) rollout_kernel(const __grid_constant__ KParams p) {
  constexpr int SP = S + 4, XS = NT + 4, NS = M::NS, HID = HD;
  constexpr int alg = ALG;
  constexpr bool WG = HD > 64;
  constexpr int HDR = 4;               // header floats: weight mbarrier
  extern __shared__ __align__(16) float smem[];
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem);
  float* part = p.partial + (size_t)blockIdx.x * p.part_stride;
  Tiles t;
  if (WG) {
    t.W = const_cast<float*>(p.blob_pol);
    t.dW = part;
    t.X = p.xbuf + (size_t)blockIdx.x * p.inp_max * XS;
    t.H1 = smem + 4;
  } else {
    t.W = smem + HDR;
    t.dW = t.W + p.w_floats;
    t.X = t.dW + p.dw_floats;
    t.H1 = t.X + p.inp_max * XS;
  }
  t.D1 = t.H1 + HID * SP;
  t.H2 = t.D1 + HID * SP;
  t.D2 = t.H2 + HID * SP;
  t.Z = t.D2 + HID * SP;      // [8][XS]: rows a (+ 4 + a: second half-stripe partial of the fused output layer)
  t.R = t.Z + 8 * XS;         // wide nets only: staging region

  const int tid = threadIdx.x;
  // column (= sample slot of the chunk) owned by this thread.  Tensor-core path: the 64 threads of warp pair p own
  // exactly the 16-sample stripes {sub * S + 16 p .. + 15} that the pair's MLP GEMMs produce, so the pair never has
  // to synchronise with the rest of the CTA outside the weight-gradient reductions.
  const int col = WG ? tid : (((tid & 63) >> 4) * S + 16 * (tid >> 6) + (tid & 15));
  auto scope_sync = [&]() {
    if (WG) __syncthreads();
    else pair_sync();
  };
// forward / backward of one sub-tile on the path this instantiation was built for
#define MLP_FWD(FULL, OUT, L, ts, Zout) mlp_forward<HD, S, NT, FULL, OUT>(L, ts, Zout)
#define MLP_BWD(WANT_DW, L, ts, want_dx) mlp_backward<HD, S, NT, WANT_DW>(L, ts, want_dx)
  const NetL& P = p.pol;
  const NetL& V = p.val;
  const int H = p.horizon, obs_dim = P.obs, TCH = p.tape_ch;
  const long long B = p.batch;
  uint32_t phase = 0;

  if (tid == 0) {
    mbar_init(mbar, 1);
    fence_mbar_init();
  }
  for (int i = tid; i < p.dw_floats; i += NT) t.dW[i] = 0.f;
  for (int i = tid; i < p.inp_max * XS; i += NT) t.X[i] = 0.f;   // pad rows of the observation tile stay zero
  for (int i = tid; i < 8 * XS; i += NT) t.Z[i] = 0.f;
  // TMA bulk copy of a packed weight blob into shared memory (all threads wait on the mbarrier)
  auto stage = [&](const float* gsrc, int floats) {
    __syncthreads();  // every reader of the previous blob is done
    if (WG) {         // wide nets: just switch the global blob the GEMMs read from
      t.W = const_cast<float*>(gsrc);
      return;
    }
    if (tid == 0) {
      fence_proxy_async();
      const uint32_t bytes = (uint32_t)floats * 4u;
      mbar_expect_tx(mbar, bytes);
      for (uint32_t off = 0; off < bytes; off += 32768u) {
        const uint32_t n = bytes - off < 32768u ? bytes - off : 32768u;
        tma_bulk_g2s(reinterpret_cast<char*>(t.W) + off, reinterpret_cast<const char*>(gsrc) + off, n, mbar);
      }
    }
    mbar_wait(mbar, phase);
    phase ^= 1u;
  };
  // coalesced read of the chunk's [n][obs_dim] rows, transposed into X (columns >= n are zero-filled)
  auto load_obs_chunk = [&](long long pos, int n, int ncols) {
    for (int idx = tid; idx < ncols * obs_dim; idx += NT) {
      const int s = idx / obs_dim, f = idx - s * obs_dim;
      t.X[f * XS + s] = s < n ? p.obs[(pos + s) * obs_dim + f] : 0.f;
    }
  };
  auto sub_tiles = [&](int sub) {
    Tiles ts = t;
    ts.X = t.X + sub * S;
    ts.Z = t.Z + sub * S;
    return ts;
  };

  stage(p.blob_pol, P.blob);

  float* tape = p.tape + (size_t)blockIdx.x * (size_t)H * TCH * NT;
  float loss_acc = 0.f, vmean_acc = 0.f, done_acc = 0.f;
  // constrained variants (pyth_veh3dofconti_errcstr, KIND 1): c = (|y_err| - tol_y, |u_err| - tol_u) of the INCOMING
  // observation of every step (pyth_veh3dofconti_errcstr_model.py:46-55); info["constraint"] is not masked at done
  constexpr float CSTR_EPS = 1e-8f;        // fhadp_interior.py:19 EPSILON
  float feas_acc = 0.f, cint_acc = 0.f;
  auto cstr_eval = [&](const float* o6, float& c_ext, float& c_lin, float& c_int, bool& infeasible) {
    const float c0 = fabsf(o6[1]) - p.cstr_y_tol, c1 = fabsf(o6[3]) - p.cstr_u_tol;
    const float p0 = fmaxf(c0, 0.f), p1 = fmaxf(c1, 0.f);
    c_ext = p0 * p0 + p1 * p1;
    c_lin = p0 + p1;
    c_int = logf(-fminf(c0, 0.f) + CSTR_EPS) + logf(-fminf(c1, 0.f) + CSTR_EPS);
    infeasible = !(c0 < 0.f) || !(c1 < 0.f);
  };
  // d(constraint cost of one step) / d(y_err, u_err), already weighted: w = gamma^k / B
  auto cstr_grad = [&](const float* o6, float w, bool feasible, float& gy, float& gu) {
    const float c0 = fabsf(o6[1]) - p.cstr_y_tol, c1 = fabsf(o6[3]) - p.cstr_u_tol;
    const float s0 = o6[1] > 0.f ? 1.f : (o6[1] < 0.f ? -1.f : 0.f), s1 = o6[3] > 0.f ? 1.f : (o6[3] < 0.f ? -1.f : 0.f);
    float d0, d1;
    if (p.cstr_mode == 1 || (p.cstr_mode == 3 && !feasible)) {
      d0 = p.cstr_coef * 2.f * fmaxf(c0, 0.f); d1 = p.cstr_coef * 2.f * fmaxf(c1, 0.f);
    } else if (p.cstr_mode == 2) {
      d0 = c0 > 0.f ? p.cstr_coef : 0.f; d1 = c1 > 0.f ? p.cstr_coef : 0.f;
    } else {      // interior, feasible sample: (1 / penalty) * d log(-c + eps) / dc = 1 / (penalty (c - eps)) for c <= 0
      d0 = c0 <= 0.f ? 1.f / (p.cstr_coef * (c0 - CSTR_EPS)) : 0.f;
      d1 = c1 <= 0.f ? 1.f / (p.cstr_coef * (c1 - CSTR_EPS)) : 0.f;
    }
    gy = w * d0 * s0;
    gu = w * d1 * s1;
  };

  // balanced contiguous sample range of this CTA, processed in chunks of NT samples
  const long long r0 = B * blockIdx.x / gridDim.x, r1 = B * (blockIdx.x + 1) / gridDim.x;
  for (long long pos = r0; pos < r1; pos += NT) {
    const int nv = (int)((r1 - pos) < NT ? (r1 - pos) : NT);
    const int nsub = (nv + S - 1) / S;
    __syncthreads();
    load_obs_chunk(pos, nv, nsub * S);
    __syncthreads();
    float st[NS];
    const bool valid = col < nv;
    const long long gs = pos + col;
    bool dn = valid ? (p.done[gs] != 0.f) : true;
    float vacc = 0.f;
    // constrained variants: discounted exterior|linear sum, interior (log) sum; SPIL: per constraint the safe-so-far flag
    // (value pass) or the running product of Phi (policy pass)
    // (one constraint: the second record stays 0, so scalar tail slot 3 reads 0)
    float cacc_a = p.cstr_mode == 4 ? 1.f : 0.f, cacc_b = M::NC == 1 ? 0.f : cacc_a;
    bool infeasible = false;
    int path = 0, spd = 0;                       // vehicle models: reference path / speed profile ids
    RefWindow<M::KIND, NT> win;
    win.base = nullptr; win.k0 = 0;
    // models with noise: this sample's draws of step k, [H][B][NZ]
    auto noise_at = [&](int k) -> const float* {
      if constexpr (M::KIND == 0 && M::NC > 0) return p.noise + ((size_t)k * B + gs) * M::NZ;
      else return nullptr;
    };
    if constexpr (M::KIND == 0) {
#pragma unroll
      for (int f = 0; f < NS; ++f) st[f] = f < obs_dim ? t.X[f * XS + col] : 0.f;
    } else {
#pragma unroll
      for (int f = 0; f < NS; ++f) st[f] = 0.f;
      if (valid) {
#pragma unroll
        for (int f = 0; f < 6; ++f) st[f] = p.state[gs * 6 + f];
      }
      if constexpr (M::KIND == 1) {
        float* er = p.ext_ref + (size_t)blockIdx.x * (size_t)(p.veh_P + 1 + H) * 4 * NT + tid;
        win.base = er;
        if (valid) {
          st[6] = p.ref_time[gs];
          path = (int)p.path_num[gs];
          spd = (int)p.u_num[gs];
        }
        for (int i = 0; i <= p.veh_P; ++i)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            er[(size_t)(i * 4 + c) * NT] = valid ? p.ref_points[(gs * (p.veh_P + 1) + i) * 4 + c] : 0.f;
      } else {
        win.base = p.reference + (size_t)(valid ? gs : 0) * p.ref_len * 4;
      }
    }

    // ================================ forward sweep ================================
    for (int k = 0; k < H; ++k) {
      if (alg == ALG_FHADP || alg == ALG_PIM) {
#pragma unroll
        for (int f = 0; f < NS; ++f) tape[(k * TCH + f) * NT + tid] = st[f];
        tape[(k * TCH + NS) * NT + tid] = dn ? 1.f : 0.f;
      }
      if (P.time_input) t.X[(P.in - 1) * XS + col] = (float)(k + 1);
      scope_sync();
      for (int sub = 0; sub < nsub; ++sub) {
        const Tiles ts = sub_tiles(sub);
        MLP_FWD(false, true, P, ts, ts.Z);
      }
      {
        float z[MAXA], a[MAXA], g[MAXA], apol[MAXA];
#pragma unroll
        for (int j = 0; j < MAXA; ++j)   // two half-stripe partials of the fused output layer
          z[j] = j < P.out ? t.Z[j * XS + col] + t.Z[(4 + j) * XS + col] : 0.f;
        if (alg == ALG_FHADP || alg == ALG_PIM) {
#pragma unroll
          for (int j = 0; j < MAXA; ++j)
            if (j < P.out) tape[(k * TCH + NS + 1 + j) * NT + tid] = z[j];
        }
        process_action(p, P.out, z, a, g, apol);
        const bool active = valid && (p.mask_at_done ? !dn : true);
        float r = 0.f;
        if constexpr (M::KIND == 1) {
          if (p.cstr_mode != 0 && valid) {
            float oc[6], ce, cl, ci;
            bool inf;
#pragma unroll
            for (int f = 0; f < 6; ++f) oc[f] = to_inner(p, f, t.X[f * XS + col]);
            if (p.cstr_mode == 4) {            // the constraints of the INCOMING observation
              const float cc[2] = {fabsf(oc[1]) - p.cstr_y_tol, fabsf(oc[3]) - p.cstr_u_tol};
              spil_track<2>(alg == ALG_PEV, cc, cacc_a, cacc_b);
            } else {
              cstr_eval(oc, ce, cl, ci, inf);
              cacc_a += (p.cstr_mode == 2 ? cl : ce) * p.gpow[k];
              cacc_b += ci * p.gpow[k];
              infeasible = infeasible || inf;
            }
          }
        }
        if constexpr (M::KIND == 0) {
          // state==obs models: `st` is the wrapper-level (outer) observation
          if (valid) {
            float c[nc_slots(M::NC)];
            wrapped_step<M>(p, obs_dim, st, a, active, r, dn, noise_at(k), c);
#pragma unroll
            for (int f = 0; f < NS; ++f)
              if (f < obs_dim) t.X[f * XS + col] = st[f];
            if constexpr (M::NC > 0) {         // the constraints of the RAW next state, frozen (done) samples included
              if (p.cstr_mode == 4) spil_track<M::NC>(alg == ALG_PEV, c, cacc_a, cacc_b);
            }
          }
        } else if (active) {
          const VehC vc = veh_const();
          float o6[6];
          if constexpr (M::KIND == 1) {
#pragma unroll
            for (int f = 0; f < 6; ++f) o6[f] = to_inner(p, f, t.X[f * XS + col]);
            r = M::reward(o6, a);
            veh_step(vc, st, a);
            st[6] = st[6] + vc.dt;
            const float tq = st[6] + p.veh_Pdt;
            float* nr = const_cast<float*>(win.base) + (size_t)(k + p.veh_P + 1) * 4 * NT;
            nr[0] = rt_x(p.rt, tq, path, spd);
            nr[NT] = rt_y(p.rt, tq, path, spd);
            nr[2 * NT] = rt_phi(p.rt, tq, path, spd);
            nr[3 * NT] = rt_u(p.rt, tq, spd);
            win.k0 = k + 1;
            veh_write_obs<M::KIND, NT>(st, win, p.veh_P, t.X + col, XS, o6);
            if (p.obs_scaling) veh_scale_obs(p, obs_dim, t.X + col, XS);
            dn = M::done(o6);
          } else {
            float q[4];
            win.k0 = p.ref_t + k;
            win.get(0, q);
            r = M::reward(st, q, a);
            veh_step(vc, st, a);
            win.k0 = p.ref_t + k + 1;
            veh_write_obs<M::KIND, NT>(st, win, p.veh_P, t.X + col, XS, o6);
            if (p.obs_scaling) veh_scale_obs(p, obs_dim, t.X + col, XS);
            win.get(0, q);
            dn = M::done(st, q);
          }
        }
        if (valid) {
          r = shape_reward(p, r);      // ShapingReward sits outside MaskAtDone: a masked sample pays (0 + shift) * scale
          vacc += r * p.gpow[k];
        }
        if (alg == ALG_TRACE && valid) {
          const size_t row = (size_t)k * B + gs;
          if (p.tr_obs)
            for (int f = 0; f < obs_dim; ++f) p.tr_obs[row * obs_dim + f] = t.X[f * XS + col];
          if (p.tr_act)
            for (int j = 0; j < P.out; ++j) p.tr_act[row * P.out + j] = apol[j];
          if (p.tr_rew) p.tr_rew[row] = r;
          if (p.tr_done) p.tr_done[row] = dn ? 1.f : 0.f;
        }
      }
    }
    if (valid && dn) done_acc += 1.f;
    float fz_y = 0.f, fz_u = 0.f;     // constrained variants: (y_err, u_err) of the observation a done sample is frozen at
    if constexpr (M::KIND == 1) {
      if (p.cstr_mode != 0) {
        fz_y = t.X[1 * XS + col]; fz_u = t.X[3 * XS + col];
        if (p.obs_scaling) { fz_y = fz_y / p.osc[1] - p.osh[1]; fz_u = fz_u / p.osc[3] - p.osh[3]; }
      }
    }
    if (alg == ALG_TRACE) continue;

    // ============================ terminal value (INFADP) ============================
    float lam[NS];
#pragma unroll
    for (int f = 0; f < NS; ++f) lam[f] = 0.f;
    if (alg != ALG_FHADP) {
      stage(p.blob_vtg, V.blob);  // leading __syncthreads also publishes X = o_n
      const float gn = p.gpow[H];
      // SPIL's value target keeps gamma^n v_target(o_n) for done samples too (spil.py:209, no (~d) mask)
      const bool term = valid && (!dn || (M::NC > 0 && p.cstr_mode == 4));
      if (alg == ALG_PIM) {
        t.Z[col] = term ? -gn * p.inv_B : 0.f;     // row 0: d loss / d v_target(o_n); rows 1 (+5) receive v
        scope_sync();
      }
      for (int sub = 0; sub < nsub; ++sub) {
        const Tiles ts = sub_tiles(sub);
        if (alg == ALG_PIM) {
          MLP_FWD(true, true, V, ts, ts.Z + XS);
          MLP_BWD(false, V, ts, true);
        } else {
          MLP_FWD(false, true, V, ts, ts.Z + XS);
        }
      }
      if (term) {
        vacc += gn * (t.Z[XS + col] + t.Z[5 * XS + col]);
        if (alg == ALG_PIM) {
          if constexpr (M::KIND == 0) {
#pragma unroll
            for (int f = 0; f < NS; ++f)
              if (f < obs_dim) lam[f] = t.X[f * XS + col];
          } else {
            // o_n = get_obs(state_n, window_n): pull the value gradient back onto the robot state
            const float zero6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            win.k0 = (M::KIND == 1 ? 0 : p.ref_t) + H;
            veh_obs_bwd<M::KIND, NT>(st, win, p.veh_P, t.X + col, XS, zero6, p.obs_scaling ? p.osc : nullptr, lam);
          }
        }
      }
    }

    if (alg == ALG_PEV) {
      if constexpr (M::NC > 0) {
        if (p.cstr_mode == 4 && valid) {     // SPIL: safe trajectories per constraint -> scalar tail slots 2 and 3
          cint_acc += cacc_a;
          feas_acc += cacc_b;
        }
      }
      // loss_v = mean((v(o_0) - backup)^2), gradient w.r.t. the value net only
      stage(p.blob_val, V.blob);
      load_obs_chunk(pos, nv, nsub * S);
      __syncthreads();
      for (int sub = 0; sub < nsub; ++sub) {
        const Tiles ts = sub_tiles(sub);
        MLP_FWD(true, true, V, ts, ts.Z + XS);
        if (col / S == sub) {
          float zb = 0.f;
          if (valid) {
            const float v0 = t.Z[XS + col] + t.Z[5 * XS + col];
            const float diff = v0 - vacc;
            loss_acc += diff * diff * p.inv_B;
            vmean_acc += v0 * p.inv_B;
            zb = 2.f * diff * p.inv_B;
          }
          t.Z[col] = zb;
        }
        scope_sync();
        MLP_BWD(true, V, ts, false);
      }
      stage(p.blob_pol, P.blob);
      continue;
    }

    float ret = vacc;                    // the per-sample objective whose negated batch mean is the loss
    if constexpr (M::NC > 0) {
      if (p.cstr_mode == 4 && valid) {
        // SPIL: loss_pi = -mean(w_r R + sum_i w_c,i prod_k Phi(c_k,i))   (spil.py:253-255); tail [1] mean R,
        // [2] / [3] mean Phi product of constraint 0 / 1
        if constexpr (M::NC == 1) ret = p.spil_w[0] * vacc + cacc_a * p.spil_w[1];
        else ret = p.spil_w[0] * vacc + (cacc_a * p.spil_w[1] + cacc_b * p.spil_w[2]);
        vmean_acc += vacc * p.inv_B;
        cint_acc += cacc_a * p.inv_B;
        feas_acc += cacc_b * p.inv_B;
      }
    }
    if (valid) loss_acc += -ret * p.inv_B;
    const bool feasible = !infeasible;
    if constexpr (M::KIND == 1) {
      if (p.cstr_mode != 0 && p.cstr_mode != 4 && valid) {
        // exterior: penalty * mean(v_c); Lagrangian: multiplier * mean(v_c);
        // interior: mean(v_int * feasible) / penalty + penalty * mean(v_ext * ~feasible)   (fhadp_interior.py:78-84)
        float cl;
        if (p.cstr_mode == 3) cl = feasible ? cacc_b / p.cstr_coef : p.cstr_coef * cacc_a;
        else cl = p.cstr_coef * cacc_a;
        loss_acc += cl * p.inv_B;
        vmean_acc += ((p.cstr_mode == 3 && feasible) ? 0.f : cacc_a) * p.inv_B;   // tb "constraint loss" (exterior part)
        if (p.cstr_mode == 3) cint_acc += feasible ? cacc_b / p.cstr_coef * p.inv_B : 0.f;
        feas_acc += feasible ? 1.f : 0.f;
      }
    }
    if (alg == ALG_PIM) stage(p.blob_pol, P.blob);

    // ================================ reverse sweep ================================
    float cbar_y = 0.f, cbar_u = 0.f;   // constrained variants: adjoint of the FROZEN observation carried to the step that made it
    for (int k = H - 1; k >= 0; --k) {
      // per-sample adjoint of step k on every thread (state, done flag and policy output come from the tape)
      if constexpr (M::KIND != 0) {
        if (k == 0) {             // step 0 consumes the caller's observation, not a re-derived one
          __syncthreads();
          load_obs_chunk(pos, nv, nsub * S);
          __syncthreads();
        }
      }
#pragma unroll
      for (int f = 0; f < NS; ++f) st[f] = tape[(k * TCH + f) * NT + tid];
      const bool dnk = tape[(k * TCH + NS) * NT + tid] != 0.f;
      float o6[6];                // vehicle models: first six observation entries of step k
      if constexpr (M::KIND == 0) {
#pragma unroll
        for (int f = 0; f < NS; ++f)
          if (f < obs_dim) t.X[f * XS + col] = st[f];
      } else {
        win.k0 = (M::KIND == 1 ? 0 : p.ref_t) + k;
        if (k > 0) {
          // only samples that were live at step k have a fully written window; the others get zeros
          // (their deltas are zero anyway, but 0 * garbage must never reach the weight gradients)
          if (valid && !(p.mask_at_done && dnk)) {
            veh_write_obs<M::KIND, NT>(st, win, p.veh_P, t.X + col, XS, o6);
            if (p.obs_scaling) {
              veh_scale_obs(p, obs_dim, t.X + col, XS);
#pragma unroll
              for (int f = 0; f < 6; ++f) o6[f] = to_inner(p, f, t.X[f * XS + col]);   // as the forward sweep saw it
            }
          } else {
            for (int f = 0; f < obs_dim; ++f) t.X[f * XS + col] = 0.f;
#pragma unroll
            for (int f = 0; f < 6; ++f) o6[f] = 0.f;
          }
        } else {
#pragma unroll
          for (int f = 0; f < 6; ++f) o6[f] = to_inner(p, f, t.X[f * XS + col]);
        }
      }
      if (P.time_input) t.X[(P.in - 1) * XS + col] = (float)(k + 1);
      const bool active = valid && (p.mask_at_done ? !dnk : true);
      // SPIL on a model whose constraints read the raw next state: a frozen (done) sample still steps, and its constraint
      // pulls back onto the action and the frozen observation
      const bool cstep = M::KIND == 0 && M::NC > 0 && p.cstr_mode == 4 && valid;
      float ro6[6];               // KIND 1: d loss / d obs_k[0..5] through the reward
#pragma unroll
      for (int f = 0; f < 6; ++f) ro6[f] = 0.f;
      {
        float zb[MAXA];
#pragma unroll
        for (int j = 0; j < MAXA; ++j) zb[j] = 0.f;
        if (active || cstep) {
          float z[MAXA], a[MAXA], g[MAXA], abar[MAXA];
#pragma unroll
          for (int j = 0; j < MAXA; ++j) z[j] = j < P.out ? tape[(k * TCH + NS + 1 + j) * NT + tid] : 0.f;
          process_action(p, P.out, z, a, g, nullptr);
          float rho = reward_adjoint(p, k);
          if constexpr (M::NC > 0) {
            if (p.cstr_mode == 4) rho *= p.spil_w[0];     // SPIL: w_r weights the return
          }
#pragma unroll
          for (int j = 0; j < MAXA; ++j) abar[j] = 0.f;
          if constexpr (M::KIND == 0) {
            // lam: adjoint of the outer observation obs_{k+1}
            if constexpr (M::NC > 0) {
              // d(-w_c / B prod_s Phi(c_s)) / dc_k = -w_c / B (prod_s Phi_s) dlog Phi(c_k)   (see the KIND 1 term below)
              const float wc = p.cstr_mode == 4 ? -p.spil_w[1] * p.inv_B * cacc_a : 0.f;
              auto cbar_of = [wc](const float* c, float* cbar) {
                float dl;
                spil_phi(c[0], dl);
                cbar[0] = wc * dl;
              };
              wrapped_step_bwd<M, MAXA, WrapRt, false>(p, obs_dim, st, a, rho, lam, abar, noise_at(k), active, cbar_of);
            } else {
              wrapped_step_bwd<M>(p, obs_dim, st, a, rho, lam, abar);
            }
          } else {
            const VehC vc = veh_const();
            veh_step_bwd(vc, st, a, lam, abar);
            if constexpr (M::KIND == 1) {
              M::reward_bwd(o6, a, rho, ro6, abar);
            } else {
              float q[4];
              win.get(0, q);
              M::reward_bwd(st, q, a, rho, lam, abar);
            }
          }
#pragma unroll
          for (int j = 0; j < MAXA; ++j) zb[j] = abar[j] * g[j];
        }
#pragma unroll
        for (int j = 0; j < MAXA; ++j)
          if (j < P.out) t.Z[j * XS + col] = zb[j];
      }
      scope_sync();
      // MLP: re-compute the hidden activations of step k per sub-tile, then back-propagate Zbar
      for (int sub = 0; sub < nsub; ++sub) {
        const Tiles ts = sub_tiles(sub);
        MLP_FWD(true, false, P, ts, nullptr);
        MLP_BWD(true, P, ts, k > 0);
      }
      if constexpr (M::KIND == 1) {
        if (p.cstr_mode != 0 && valid && k > 0) {
          // The constraint of step k reads obs_k.  obs_k was MADE by step k - 1 iff the sample was live there (MaskAtDone
          // freezes the observation afterwards): then its adjoint (this step's + the carry of the frozen copies) goes
          // through get_obs onto state_k; else obs_k is a copy of obs_{k-1} and the adjoint is carried on.
          const bool made_here = p.mask_at_done ? tape[((k - 1) * TCH + NS) * NT + tid] == 0.f : true;
          const bool live = !(p.mask_at_done && dnk);
          float oc[6] = {0.f, live ? o6[1] : fz_y, 0.f, live ? o6[3] : fz_u, 0.f, 0.f};
          float gy, gu;
          if (p.cstr_mode == 4) {
            // SPIL: d(-w_c,i / B prod_s Phi(c_s,i)) / dc_k,i = -w_c,i / B (prod_s Phi_s,i) dlog Phi(c_k,i); Phi >= 0.188, so
            // the product over s != k is the total product over Phi_k
            float d0, d1;
            spil_phi(fabsf(oc[1]) - p.cstr_y_tol, d0);
            spil_phi(fabsf(oc[3]) - p.cstr_u_tol, d1);
            const float s0 = oc[1] > 0.f ? 1.f : (oc[1] < 0.f ? -1.f : 0.f), s1 = oc[3] > 0.f ? 1.f : (oc[3] < 0.f ? -1.f : 0.f);
            gy = -p.spil_w[1] * p.inv_B * cacc_a * d0 * s0;
            gu = -p.spil_w[2] * p.inv_B * cacc_b * d1 * s1;
          } else {
            cstr_grad(oc, p.gpow[k] * p.inv_B, feasible, gy, gu);
          }
          gy += cbar_y; gu += cbar_u;
          if (made_here) {
            cbar_y = cbar_u = 0.f;
            if (active) {
              ro6[1] += gy; ro6[3] += gu;      // joins the reward's observation adjoint in veh_obs_bwd below
            } else {                           // done AT step k - 1: only the constraint looks at this observation
              const float e6[6] = {0.f, gy, 0.f, gu, 0.f, 0.f};
              veh_obs_bwd<M::KIND, NT>(st, win, p.veh_P, t.X + col, XS, e6, p.obs_scaling ? p.osc : nullptr, lam);
            }
          } else {
            cbar_y = gy; cbar_u = gu;
          }
        }
      }
      if ((active || cstep) && k > 0) {
        if constexpr (M::KIND == 0) {
#pragma unroll
          for (int f = 0; f < NS; ++f)
            if (f < obs_dim) lam[f] += t.X[f * XS + col];
        } else {
          veh_obs_bwd<M::KIND, NT>(st, win, p.veh_P, t.X + col, XS, ro6, p.obs_scaling ? p.osc : nullptr, lam);
        }
      }
    }
  }

  // ============================ per-CTA partials ============================
  __syncthreads();
  const int nparam = (alg == ALG_PEV) ? V.nparam : P.nparam;
  if (alg != ALG_TRACE && !WG) {
    const NetL& U = (alg == ALG_PEV) ? V : P;
    for (int i = tid; i < nparam; i += NT) {      // accumulator layout -> torch flat layout
      int j;
      if (i < U.g_w2) j = i;                                                    // W1, b1 (offsets coincide)
      else if (i < U.g_b2) { const int q = i - U.g_w2; j = U.d_w2 + (q / HID) * U.ldw2 + (q % HID); }
      else j = i - U.g_b2 + U.d_b2;                                             // b2, W3, b3
      part[i] = t.dW[j];
    }
  }
  // block reduction of the three scalars (fixed order)
  float* red = t.H1;  // free at this point, HID*(S+4) >= 3*NT floats
  red[tid] = loss_acc;
  red[NT + tid] = vmean_acc;
  // interior point: the weighted log-barrier term; SPIL: safe count / mean Phi product of constraint 0
  red[2 * NT + tid] = p.cstr_mode >= 3 ? cint_acc : done_acc;
  __syncthreads();
  if (tid < 3) {
    float s = 0.f;
    for (int i = 0; i < NT; ++i) s += red[tid * NT + i];
    part[nparam + tid] = s;
  }
  __syncthreads();
  red[tid] = feas_acc;              // constrained variants: number of feasible samples (slot 3 of the scalar tail); SPIL: constraint 1
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
    for (int i = 0; i < NT; ++i) s += red[i];
    part[nparam + 3] = s;
  }
#undef MLP_FWD
#undef MLP_BWD
}

// Batched inference of one MLP (policy with tanh squashing when `squash`, else raw value output)
template <int HD, int S, int NT>
__global__ void __launch_bounds__(NT, 1) mlp_infer_kernel(const __grid_constant__ KParams p, const float* blob, int use_val,
                                                          const float* __restrict__ obs, long long B, float virtual_t,
                                                          int squash, float* __restrict__ out) {
  constexpr int SP = S + 4, XS = NT + 4, HID = HD;
  constexpr bool WG = HD > 64;
  extern __shared__ __align__(16) float smem[];
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem);
  const NetL& L = use_val ? p.val : p.pol;
  Tiles t;
  if (WG) {
    t.W = const_cast<float*>(blob);
    t.X = p.xbuf + (size_t)blockIdx.x * p.inp_max * XS;
    t.H1 = smem + 4;
  } else {
    t.W = smem + 4;
    t.X = t.W + p.w_floats;
    t.H1 = t.X + p.inp_max * XS;
  }
  for (int i = threadIdx.x; i < p.inp_max * XS; i += NT) t.X[i] = 0.f;
  t.dW = nullptr;
  t.D1 = t.H1;
  t.H2 = t.H1 + HID * SP;
  t.D2 = t.H2;
  t.Z = t.H2 + HID * SP;
  t.R = t.Z + 8 * XS;
  for (int i = threadIdx.x; i < 8 * XS; i += NT) t.Z[i] = 0.f;
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(mbar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (!WG) {
    if (tid == 0) {
      fence_proxy_async();
      const uint32_t bytes = (uint32_t)L.blob * 4u;
      mbar_expect_tx(mbar, bytes);
      for (uint32_t off = 0; off < bytes; off += 32768u) {
        const uint32_t n = bytes - off < 32768u ? bytes - off : 32768u;
        tma_bulk_g2s(reinterpret_cast<char*>(t.W) + off, reinterpret_cast<const char*>(blob) + off, n, mbar);
      }
    }
    mbar_wait(mbar, 0);
  }
  const long long n_chunks = (B + NT - 1) / NT;
  for (long long c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const long long base = c * NT;
    const int nv = (int)((B - base) < NT ? (B - base) : NT);
    const int nsub = (nv + S - 1) / S;
    __syncthreads();
    for (int idx = tid; idx < nsub * S * L.obs; idx += NT) {
      const int s = idx / L.obs, f = idx - s * L.obs;
      t.X[f * XS + s] = s < nv ? obs[(base + s) * L.obs + f] : 0.f;
    }
    if (L.time_input) t.X[(L.in - 1) * XS + tid] = virtual_t;
    __syncthreads();
    for (int sub = 0; sub < nsub; ++sub) {
      Tiles ts = t;
      ts.X = t.X + sub * S;
      ts.Z = t.Z + sub * S;
      mlp_forward<HD, S, NT, false, true>(L, ts, ts.Z);
    }
    __syncthreads();
    if (tid < nv) {
      for (int j = 0; j < L.out; ++j) {
        float z = t.Z[j * XS + tid] + t.Z[(4 + j) * XS + tid];
        if (squash) z = __fadd_rn(__fmul_rn(p.pol_half[j], tanhf(z)), p.pol_mid[j]);
        out[(base + tid) * L.out + j] = z;
      }
    }
  }
}

// One wrapped-model step for explicit actions: envmodel.forward(obs, action, done, info) of the
// reference wrapper chain (create_env_model.py:104-126) for state==obs models.
template <class M>
__global__ void model_step_kernel(const __grid_constant__ KParams p, const float* __restrict__ action, int act_dim,
                                  float* __restrict__ next_obs, float* __restrict__ reward,
                                  float* __restrict__ next_done) {
  constexpr int NS = M::NS;
  const long long gs = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gs >= p.batch) return;
  const int obs_dim = p.pol.obs;
  float st[NS], a[MAXA];
#pragma unroll
  for (int f = 0; f < NS; ++f) st[f] = f < obs_dim ? p.obs[gs * obs_dim + f] : 0.f;
#pragma unroll
  for (int j = 0; j < MAXA; ++j) {
    float gg = 1.f;
    a[j] = j < act_dim ? wrap_action(p, j, action[gs * act_dim + j], gg) : 0.f;
  }
  bool dn = p.done[gs] != 0.f;
  float r = 0.f, c[nc_slots(M::NC)];
  const float* nz = nullptr;
  if constexpr (M::NC > 0) nz = p.noise + (size_t)gs * M::NZ;
  wrapped_step<M>(p, obs_dim, st, a, !(p.mask_at_done && dn), r, dn, nz, c);     // a masked sample stays done
  if constexpr (M::NC > 0) {
    if (p.cstr_out)
      for (int i = 0; i < M::NC; ++i) p.cstr_out[gs * M::NC + i] = c[i];
  }
  r = shape_reward(p, r);
  for (int f = 0; f < obs_dim; ++f) next_obs[gs * obs_dim + f] = st[f];
  reward[gs] = r;
  next_done[gs] = dn ? 1.f : 0.f;
}


// envmodel.forward(obs, action, done, info) for the vehicle models (one thread per sample, global memory only).
// Mirrors Veh3dofcontiModel.forward (pyth_veh3dofconti_model.py:91-145) / EnvModel.forward
// (env_gen_ocp/env_model/pyth_base_model.py:109-119) inside the wrapper chain: `info` is advanced even for masked
// (done) samples, exactly like the reference (MaskAtDone does not touch next_info).
template <int KIND>
__global__ void veh_step_kernel(const __grid_constant__ KParams p, const float* __restrict__ action,
                                float* __restrict__ next_obs, float* __restrict__ reward, float* __restrict__ next_done,
                                float* __restrict__ next_state, float* __restrict__ next_ref_points,
                                float* __restrict__ next_ref_time) {
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
  float r;
  bool md;
  if (KIND == 1) {
    float o[6];
#pragma unroll
    for (int f = 0; f < 6; ++f) o[f] = to_inner(p, f, obs[f]);
    r = ModelVehConti::reward(o, a);
    veh_step(vc, s, a);
    const float nt = p.ref_time[gs] + vc.dt, tq = nt + p.veh_Pdt;
    const int path = (int)p.path_num[gs], spd = (int)p.u_num[gs];
    const float* rp = p.ref_points + gs * (P + 1) * 4;
    float* nrp = next_ref_points + gs * (P + 1) * 4;
    for (int i = 0; i < P; ++i)
#pragma unroll
      for (int c = 0; c < 4; ++c) nrp[i * 4 + c] = rp[(i + 1) * 4 + c];
    nrp[P * 4 + 0] = rt_x(p.rt, tq, path, spd);
    nrp[P * 4 + 1] = rt_y(p.rt, tq, path, spd);
    nrp[P * 4 + 2] = rt_phi(p.rt, tq, path, spd);
    nrp[P * 4 + 3] = rt_u(p.rt, tq, spd);
    next_ref_time[gs] = nt;
    RefWindow<2, 1> w;             // sample-major [P+1][4] window in global memory
    w.base = nrp; w.k0 = 0;
    float o6[6];
    veh_write_obs<2, 1>(s, w, P, nobs, 1, o6);
    md = ModelVehConti::done(o6);
  } else {
    RefWindow<2, 1> w;
    w.base = p.reference + gs * (size_t)p.ref_len * 4; w.k0 = p.ref_t;
    float q[4];
    w.get(0, q);
    r = ModelVehTrack::reward(s, q, a);
    veh_step(vc, s, a);
    w.k0 = p.ref_t + 1;
    float o6[6];
    veh_write_obs<2, 1>(s, w, P, nobs, 1, o6);
    w.get(0, q);
    md = ModelVehTrack::done(s, q);
  }
#pragma unroll
  for (int f = 0; f < 6; ++f) next_state[gs * 6 + f] = s[f];
  if (p.mask_at_done && dn) {     // MaskAtDone: frozen (inner) observation, zero reward
    r = 0.f;
    for (int f = 0; f < obs_dim; ++f) nobs[f] = to_inner(p, f, obs[f]);
  }
  if (p.mask_at_done) md = md || dn;
  r = shape_reward(p, r);
  if (p.obs_scaling) veh_scale_obs(p, obs_dim, nobs, 1);
  reward[gs] = r;
  next_done[gs] = md ? 1.f : 0.f;
}

}  // namespace gops
