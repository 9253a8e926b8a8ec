// Fused rollout + loss + gradient kernel for hidden width 64 (sm_90a): shared-memory tile primitives.
//
// One CTA owns chunks of NT samples (one per thread) for the whole horizon:
//   * per-sample model state lives in the registers of its thread for all H steps;
//   * MLP weights are staged ONCE per CTA into shared memory by the TMA bulk-copy engine;
//   * MLP activations live in shared memory, feature-major [feature][sample] so that every
//     dense layer is a CTA-level GEMM with float4 shared-memory operands and FP32 FFMA;
//   * the reverse sweep re-computes the MLP activations per step from a small state tape
//     (per-CTA scratch, L2 resident) and accumulates weight gradients in shared memory;
//   * each CTA writes one gradient partial; a second kernel reduces partials in fixed order
//     (deterministic, no float atomics).
// The dense primitives are deliberately NOT inlined: the hot loop must stay I-cache resident
// (v1 inlined everything: 68k SASS instructions, `no_instruction` was the top stall).
#pragma once
#include "common.cuh"
#include "mma_tiles.cuh"

namespace gops {

// Hidden width HD is a template parameter of every primitive (64: everything in shared memory; 256: weights,
// weight-gradient accumulators and the observation tile live in global memory / L2, activations in smem).
// k-major weight tiles have row stride hp_of(HD): HD + 4 for the FFMA path (bank skew 4 for the transposed
// reads), 72 for the 64-wide tensor-core path (bank skew 8: conflict-free B-fragment loads of the forward GEMMs).
__host__ __device__ constexpr int hp_of(int HD) { return HD == 64 ? 72 : HD + 4; }

// Reference-trajectory constants as fp32 values derived on the host in double precision.
struct RtC {
  float sine_A, sine_omega, sine_phi;
  float dl_t1, dl_t2, dl_t3, dl_t4, dl_y1, dl_y2, dl_k1, dl_k2;   // k1 = (y2-y1)/(t2-t1), k2 = (y1-y2)/(t4-t3)
  float tri_k1, tri_k2, tri_T, tri_half;                         // 2A/T, -2A/T, T, T/2
  float circ_r;
  float sp_A, sp_omega, sp_phi, sp_b, sp_c1, sp_c3, sp_const;    // c1 = -A/omega, c3 = A/omega*cos(phi)
};

// Layout of one network (host computed).
struct NetL {
  int in;          // input rows incl. time column
  int inp;         // in rounded up to 4
  int obs;         // rows fed from the observation (= in - time_input)
  int out;         // outputs (<= MAXA)
  int hact, oact, time_input;
  // packed weight blob offsets (floats); blob is what TMA copies to shared memory
  //   w1: [in][HP]  (W1^T, k-major)   w2: [HID][HP] (W2^T)   w3: [out][HID]   b1,b2: [HID]   b3: [4]
  int o_w1, o_w2, o_w3, o_b1, o_b2, o_b3, blob;
  int o_w1l, o_w2l;   // 64-wide path: lo planes of the 3xTF32 split (o_w1 / o_w2 then hold the hi planes)
  int in8;            // in rounded up to 8 (k extent of the layer-1 tensor-core GEMM)
  // torch flat parameter offsets
  int g_w1, g_b1, g_w2, g_b2, g_w3, g_b3, nparam;
  // accumulator layout in shared memory (= torch layout except that W2 rows are padded to ldw2 floats so that the
  // fragment-wise read-modify-write of dw_accum_mma is not an 8-way bank conflict)
  int d_w1, d_b1, d_w2, d_b2, d_w3, d_b3, ldw2, nacc;
};

struct KParams {
  int alg, horizon, n_tiles;
  long long batch;
  float gamma, inv_B;
  const float* gpow;       // fp32(gamma^k), k = 0..H (host-computed in double like python's gamma ** k)
  NetL pol, val;
  const float* blob_pol;
  const float* blob_val;   // v        (INFADP_VALUE)
  const float* blob_vtg;   // v_target (INFADP_*)
  // inputs
  const float* obs;
  const float* done;
  const float* state;
  const float* ref_points;
  const float* path_num;
  const float* u_num;
  const float* ref_time;
  const float* reference;
  int ref_t, ref_len, veh_P;
  float veh_Pdt;           // fp32(pre_horizon * dt) as formed by the reference in python doubles
  // scratch
  float* tape;             // [grid][H][tape_ch][NT]  (state, done flag, then per policy output: mma.sync the pre-activation
                           // z; wgmma the action a and d a / d z)
  int tape_ch;
  float* ext_ref;          // veh3dofconti: [grid][P+1+H][4][NT] raw reference points (window slides by one per step)
  float* partial;          // [grid][part_stride]
  float* xbuf;             // wide nets: [grid][inp_max][NT+4] observation tile in global memory
  int hid;                 // hidden width of both networks (64 or 256)
  int part_stride;
  // smem carve (floats)
  int w_floats, dw_floats, inp_max;
  // trace outputs (alg == ALG_TRACE)
  float* tr_obs; float* tr_act; float* tr_rew; float* tr_done;
  // constrained FHADP variants (fhadp_exterior / fhadp_lagrangian / fhadp_interior.py): 0 none, 1 exterior penalty,
  // 2 Lagrangian, 3 interior point, 4 SPIL (spil.py: safe-trajectory counts on the value pass, the weighted
  // Phi-product term on the policy pass); cstr_coef = penalty / multiplier; tolerances of the error-constraint model
  int cstr_mode;
  float cstr_coef, cstr_y_tol, cstr_u_tol;
  const float* spil_w;     // cstr_mode 4, policy pass: device [w_r, w_c0, w_c1] written by the SPIL controller kernel
  // models with noise (pyth_mobilerobot): device draws, [H][B][2] per rollout / [B][2] per model step; the model step's
  // [B][NC] constraints out (gops_b200_plan_set_model_io)
  const float* noise;
  float* cstr_out;
  // env_gen_ocp veh3dof_tracking_detour (lw_detour.cuh): surrounding-vehicle predictions [B][surr_len][1][5] (x, y, phi, u,
  // delta), circle offset d = (length - width) / 2 and 2 r = width of the bicircle collision model
  int veh_detour, surr_len;
  const float* surr;
  float veh_dc, veh_2r;
  // reward r = -veh_rscale * sum_i veh_rc[i] * (ex, ey, ephi, eu, w, steer, a_x)_i^2 + veh_roff; lateral termination bound
  float veh_rscale, veh_roff, veh_rc[7], veh_ydone;
  // wrappers
  int action_scale, clip_action, clip_obs, mask_at_done, reward_shaping;
  float reward_shift, reward_scale;
  int obs_scaling, repeat_num, sum_reward;   // ScaleObservation / ActionRepeat (repeat_num 0 = absent)
  const float* osc;        // device arrays [obs_dim]: observation scale / shift
  const float* osh;
  float min_action[MAXA], max_action[MAXA], act_low[MAXA], act_high[MAXA];
  float pol_half[MAXA], pol_mid[MAXA];
  float obs_low[kMaxObs], obs_high[kMaxObs];   // ClipObservation bounds of the state==obs models
  // LQ
  int lq_n, lq_m;
  float lq_inv_IA[LQN * LQN], lq_B[LQN * MAXA], lq_Q[LQN], lq_R[MAXA];
  float lq_dt, lq_rs, lq_rsh;
  RtC rt;
};

constexpr int ALG_FHADP = GOPS_ALG_FHADP, ALG_PIM = GOPS_ALG_INFADP_POLICY, ALG_PEV = GOPS_ALG_INFADP_VALUE,
              ALG_TRACE = 3;

// cp.async (LDGSTS) helpers for the wide-net path: weight k-slices are staged global -> shared, double buffered
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Warp tiling of a [HID x S] output tile: every warp is 4 (feature) x 8 (sample) threads, a thread
// owns TM features x 4 samples.  One k-step then needs ONE 64 B and ONE 128 B shared wavefront per warp.
template <int HD, int S, int NT>
struct Map {
  static constexpr int HID = HD, HP = hp_of(HD);
  static constexpr int SP = S + 4, NW = NT / 32, WN = S / 32, WM = NW / WN, TM = HID / (4 * WM);
  static_assert(S % 32 == 0 && NW % WN == 0 && WM >= 1 && TM >= 1 && TM * 4 * WM == HID && TM % 4 == 0, "bad tiling");
  int n0, mt;   // first sample column, feature-thread index (0 .. 4*WM-1)
  __device__ __forceinline__ Map() {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    n0 = ((w % WN) * 8 + (l & 7)) * 4;
    mt = (w / WN) * 4 + (l >> 3);
  }
};

// ---------------------------------------------------------------------------------------------
// P[m][n] = bias[m] + sum_k A[k][m] * B[k][n]   (pre-activations of a hidden layer)
// A: k-major weights [K][HP], B: [K][SP].  Thread owns CONTIGUOUS features m0 .. m0+TM-1.
// ---------------------------------------------------------------------------------------------
template <int HD, int S, int NT>
__device__ __noinline__ void gemm_fwd(const float* __restrict__ A, const float* __restrict__ Bm, int ldb, int K,
                                      const float* __restrict__ bias, float* __restrict__ P) {
  using M = Map<HD, S, NT>;
  constexpr int HID = HD, HP = hp_of(HD);
  constexpr int SP = M::SP, TM = M::TM;
  const M mp;
  const int m0 = mp.mt * TM;
  float acc[TM][4];
#pragma unroll
  for (int j = 0; j < TM; ++j) {
    const float bb = bias[m0 + j];
    acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = bb;
  }
  const float* bp = Bm + mp.n0;
  const float* ap = A + m0;
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    const float4 b = *reinterpret_cast<const float4*>(bp + k * ldb);
    float a[TM];
#pragma unroll
    for (int q = 0; q < TM / 4; ++q) {
      const float4 av = *reinterpret_cast<const float4*>(ap + k * HP + 4 * q);
      a[4 * q] = av.x; a[4 * q + 1] = av.y; a[4 * q + 2] = av.z; a[4 * q + 3] = av.w;
    }
#pragma unroll
    for (int j = 0; j < TM; ++j) {
      acc[j][0] = fmaf(a[j], b.x, acc[j][0]);
      acc[j][1] = fmaf(a[j], b.y, acc[j][1]);
      acc[j][2] = fmaf(a[j], b.z, acc[j][2]);
      acc[j][3] = fmaf(a[j], b.w, acc[j][3]);
    }
  }
#pragma unroll
  for (int j = 0; j < TM; ++j)
    *reinterpret_cast<float4*>(P + (m0 + j) * SP + mp.n0) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
}

// In-place activation of the tile a thread just wrote with gemm_fwd (same ownership -> no barrier):
// H <- act(P); if D != nullptr also D <- act'(P).  Rolled loop: the activation code exists once.
template <int HD, int S, int NT>
__device__ __noinline__ void act_pass(float* __restrict__ H, float* __restrict__ D, int act) {
  using M = Map<HD, S, NT>;
  constexpr int HID = HD, HP = hp_of(HD);
  constexpr int SP = M::SP, TM = M::TM;
  const M mp;
  const int m0 = mp.mt * TM;
#pragma unroll 1
  for (int j = 0; j < TM; ++j) {
    float* hp = H + (m0 + j) * SP + mp.n0;
    const float4 p = *reinterpret_cast<const float4*>(hp);
    float4 h, d;
    if (D != nullptr) {
      act_fwd_grad(act, p.x, h.x, d.x); act_fwd_grad(act, p.y, h.y, d.y);
      act_fwd_grad(act, p.z, h.z, d.z); act_fwd_grad(act, p.w, h.w, d.w);
      *reinterpret_cast<float4*>(D + (m0 + j) * SP + mp.n0) = d;
    } else {
      h.x = act_fwd(act, p.x); h.y = act_fwd(act, p.y); h.z = act_fwd(act, p.z); h.w = act_fwd(act, p.w);
    }
    *reinterpret_cast<float4*>(hp) = h;
  }
}

// ---------------------------------------------------------------------------------------------
// D[i][n] <- D[i][n] * sum_o A[i][o] * Dl[o][n]     (delta of a hidden layer, in place over D)
// A: the SAME k-major tile [HID][HP] read transposed; thread owns INTERLEAVED rows i = mt + 4*WM*j so
// the four feature-threads of a warp read consecutive rows (HP = 68 -> banks skewed by 4, conflict-free).
// ---------------------------------------------------------------------------------------------
template <int HD, int S, int NT>
__device__ __noinline__ void gemm_bwd(const float* __restrict__ A, const float* __restrict__ Dl,
                                      float* __restrict__ D) {
  using M = Map<HD, S, NT>;
  constexpr int HID = HD, HP = hp_of(HD);
  constexpr int SP = M::SP, TM = M::TM, RS = 4 * M::WM;
  const M mp;
  float acc[TM][4];
#pragma unroll
  for (int j = 0; j < TM; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  const float* ap = A + mp.mt * HP;
  const float* bp = Dl + mp.n0;
#pragma unroll 2
  for (int o = 0; o < HID; o += 4) {
    float4 b[4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) b[kk] = *reinterpret_cast<const float4*>(bp + (o + kk) * SP);
#pragma unroll
    for (int j = 0; j < TM; ++j) {
      const float4 a = *reinterpret_cast<const float4*>(ap + j * RS * HP + o);
      acc[j][0] = fmaf(a.x, b[0].x, acc[j][0]); acc[j][1] = fmaf(a.x, b[0].y, acc[j][1]);
      acc[j][2] = fmaf(a.x, b[0].z, acc[j][2]); acc[j][3] = fmaf(a.x, b[0].w, acc[j][3]);
      acc[j][0] = fmaf(a.y, b[1].x, acc[j][0]); acc[j][1] = fmaf(a.y, b[1].y, acc[j][1]);
      acc[j][2] = fmaf(a.y, b[1].z, acc[j][2]); acc[j][3] = fmaf(a.y, b[1].w, acc[j][3]);
      acc[j][0] = fmaf(a.z, b[2].x, acc[j][0]); acc[j][1] = fmaf(a.z, b[2].y, acc[j][1]);
      acc[j][2] = fmaf(a.z, b[2].z, acc[j][2]); acc[j][3] = fmaf(a.z, b[2].w, acc[j][3]);
      acc[j][0] = fmaf(a.w, b[3].x, acc[j][0]); acc[j][1] = fmaf(a.w, b[3].y, acc[j][1]);
      acc[j][2] = fmaf(a.w, b[3].z, acc[j][2]); acc[j][3] = fmaf(a.w, b[3].w, acc[j][3]);
    }
  }
#pragma unroll
  for (int j = 0; j < TM; ++j) {
    float* dp = D + (mp.mt + j * RS) * SP + mp.n0;
    float4 d = *reinterpret_cast<const float4*>(dp);
    d.x *= acc[j][0]; d.y *= acc[j][1]; d.z *= acc[j][2]; d.w *= acc[j][3];
    *reinterpret_cast<float4*>(dp) = d;
  }
}

// Z[a][s] = b3[a] + sum_i W3[a][i] * H[i][s]       (output layer, out <= MAXA)
template <int HD, int S, int NT>
__device__ __noinline__ void out_layer(const float* __restrict__ W3, const float* __restrict__ b3,
                                       const float* __restrict__ H, int out, float* __restrict__ Z, int ldz) {
  constexpr int SP = S + 4, HID = HD;
  for (int idx = threadIdx.x; idx < out * S; idx += NT) {
    const int a = idx / S, s = idx - a * S;
    float a0 = b3[a], a1 = 0.f;
#pragma unroll 8
    for (int i = 0; i < HID; i += 2) {
      a0 = fmaf(W3[a * HID + i], H[i * SP + s], a0);
      a1 = fmaf(W3[a * HID + i + 1], H[(i + 1) * SP + s], a1);
    }
    Z[a * ldz + s] = a0 + a1;
  }
}

// D[i][s] <- D[i][s] * sum_a W3[a][i] * Zb[a][s]   (delta of the last hidden layer, in place)
template <int HD, int S, int NT>
__device__ __noinline__ void delta_from_out(const float* __restrict__ W3, const float* __restrict__ Zb, int ldz, int out,
                                            float* __restrict__ D) {
  using M = Map<HD, S, NT>;
  constexpr int HID = HD, HP = hp_of(HD);
  constexpr int SP = M::SP, TM = M::TM;
  const M mp;
  const int m0 = mp.mt * TM;
  float4 zb[MAXA];
#pragma unroll
  for (int a = 0; a < MAXA; ++a)
    zb[a] = a < out ? *reinterpret_cast<const float4*>(Zb + a * ldz + mp.n0) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
  for (int j = 0; j < TM; ++j) {
    const int row = m0 + j;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int a = 0; a < MAXA; ++a)
      if (a < out) {
        const float w = W3[a * HID + row];
        acc.x = fmaf(w, zb[a].x, acc.x); acc.y = fmaf(w, zb[a].y, acc.y);
        acc.z = fmaf(w, zb[a].z, acc.z); acc.w = fmaf(w, zb[a].w, acc.w);
      }
    float4 d = *reinterpret_cast<const float4*>(D + row * SP + mp.n0);
    d.x *= acc.x; d.y *= acc.y; d.z *= acc.z; d.w *= acc.w;
    *reinterpret_cast<float4*>(D + row * SP + mp.n0) = d;
  }
}

// dst[o][i] += sum_s Dl[o][s] * Xl[i][s]   for o < RO, i < RI   (weight gradient; dst row stride ld)
// Tiles own interleaved rows (o = to + tiles_o*j) so that lanes of a warp touch consecutive rows
// of the (S+4)-strided tiles -> conflict-free float4 shared loads.
template <int HD, int S, int NT, int TO, int TI>
__device__ __noinline__ void dw_accum(const float* __restrict__ Dl, int ldd, int RO, const float* __restrict__ Xl,
                                      int ldx, int RI, float* __restrict__ dst, int ld, int toff = 0,
                                      bool swz_x = false) {
  const int tiles_o = (RO + TO - 1) / TO, tiles_i = (RI + TI - 1) / TI;
  for (int tile = (threadIdx.x + NT - (toff % NT)) % NT; tile < tiles_o * tiles_i; tile += NT) {
    const int ti = tile % tiles_i, to = tile / tiles_i;
    float acc[TO][TI];
#pragma unroll
    for (int j = 0; j < TO; ++j)
#pragma unroll
      for (int q = 0; q < TI; ++q) acc[j][q] = 0.f;
    const float* dp[TO];
    const float* xp[TI];
    int swx[TI];      // activation-tile swizzle: odd rows are stored with column ^ 8
#pragma unroll
    for (int j = 0; j < TO; ++j) dp[j] = Dl + min(to + tiles_o * j, RO - 1) * ldd;
#pragma unroll
    for (int q = 0; q < TI; ++q) {
      const int row = min(ti + tiles_i * q, RI - 1);
      xp[q] = Xl + row * ldx;
      swx[q] = swz_x ? (row & 1) << 3 : 0;
    }
#pragma unroll 2
    for (int s = 0; s < S; s += 4) {
      float4 d[TO], x[TI];
#pragma unroll
      for (int j = 0; j < TO; ++j) d[j] = *reinterpret_cast<const float4*>(dp[j] + s);
#pragma unroll
      for (int q = 0; q < TI; ++q) x[q] = *reinterpret_cast<const float4*>(xp[q] + (s ^ swx[q]));
#pragma unroll
      for (int j = 0; j < TO; ++j)
#pragma unroll
        for (int q = 0; q < TI; ++q) {
          acc[j][q] = fmaf(d[j].x, x[q].x, acc[j][q]);
          acc[j][q] = fmaf(d[j].y, x[q].y, acc[j][q]);
          acc[j][q] = fmaf(d[j].z, x[q].z, acc[j][q]);
          acc[j][q] = fmaf(d[j].w, x[q].w, acc[j][q]);
        }
    }
#pragma unroll
    for (int j = 0; j < TO; ++j) {
      const int o = to + tiles_o * j;
#pragma unroll
      for (int q = 0; q < TI; ++q) {
        const int i = ti + tiles_i * q;
        if (o < RO && i < RI) dst[o * ld + i] += acc[j][q];
      }
    }
  }
}

// dst[o] += sum_s Dl[o][s]        (bias gradient)
template <int HD, int S, int NT>
__device__ __noinline__ void rowsum_accum(const float* __restrict__ Dl, int ldd, int RO, float* __restrict__ dst,
                                          int toff = 0) {
  for (int o = (threadIdx.x + NT - (toff % NT)) % NT; o < RO; o += NT) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 4
    for (int s = 0; s < S; s += 4) {
      const float4 d = *reinterpret_cast<const float4*>(Dl + o * ldd + s);
      a0 += d.x; a1 += d.y; a2 += d.z; a3 += d.w;
    }
    dst[o] += (a0 + a1) + (a2 + a3);
  }
}

// Xb[i][s] = sum_o W1k[i][o] * Dl[o][s]  for i < M (M <= 8*MG)   (input gradient; W1k: [in][HP] k-major)
template <int HD, int S, int NT>
__device__ __noinline__ void gemm_dx(const float* __restrict__ W1k, const float* __restrict__ W1lo,
                                     const float* __restrict__ Dl, int M, float* __restrict__ Xb, int ldx) {
  constexpr int SP = S + 4, NTN = S / 4, MG = NT / NTN, JM = 8, HID = HD, HP = hp_of(HD);
  const int tid = threadIdx.x, nt = tid % NTN, mg = tid / NTN;
  const int J = (M - mg + MG - 1) / MG;  // rows mg, mg+MG, ... < M
  if (J <= 0) return;
  float acc[JM][4];
#pragma unroll
  for (int j = 0; j < JM; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll 1
  for (int o = 0; o < HID; o += 4) {
    float4 d[4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) d[kk] = *reinterpret_cast<const float4*>(Dl + (o + kk) * SP + 4 * nt);
#pragma unroll
    for (int j = 0; j < JM; ++j)
      if (j < J) {
        float4 w = *reinterpret_cast<const float4*>(W1k + (mg + MG * j) * HP + o);
        if (W1lo != nullptr) {   // hi + lo == the fp32 weight exactly
          const float4 wl = *reinterpret_cast<const float4*>(W1lo + (mg + MG * j) * HP + o);
          w.x += wl.x; w.y += wl.y; w.z += wl.z; w.w += wl.w;
        }
        acc[j][0] = fmaf(w.x, d[0].x, acc[j][0]); acc[j][1] = fmaf(w.x, d[0].y, acc[j][1]);
        acc[j][2] = fmaf(w.x, d[0].z, acc[j][2]); acc[j][3] = fmaf(w.x, d[0].w, acc[j][3]);
        acc[j][0] = fmaf(w.y, d[1].x, acc[j][0]); acc[j][1] = fmaf(w.y, d[1].y, acc[j][1]);
        acc[j][2] = fmaf(w.y, d[1].z, acc[j][2]); acc[j][3] = fmaf(w.y, d[1].w, acc[j][3]);
        acc[j][0] = fmaf(w.z, d[2].x, acc[j][0]); acc[j][1] = fmaf(w.z, d[2].y, acc[j][1]);
        acc[j][2] = fmaf(w.z, d[2].z, acc[j][2]); acc[j][3] = fmaf(w.z, d[2].w, acc[j][3]);
        acc[j][0] = fmaf(w.w, d[3].x, acc[j][0]); acc[j][1] = fmaf(w.w, d[3].y, acc[j][1]);
        acc[j][2] = fmaf(w.w, d[3].z, acc[j][2]); acc[j][3] = fmaf(w.w, d[3].w, acc[j][3]);
      }
  }
#pragma unroll
  for (int j = 0; j < JM; ++j)
    if (j < J)
      *reinterpret_cast<float4*>(Xb + (mg + MG * j) * ldx + 4 * nt) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
}

// ---------------------------------------------------------------------------------------------
// Wide nets (HD = 256): the weights live in global memory (L2); the GEMMs stream them through shared memory in
// double-buffered k-slices (cp.async), so the inner loops read shared memory only.
// ---------------------------------------------------------------------------------------------
// P[m][n] = bias[m] + sum_k A[k][m] * B[k][n];  A: global [K][HP];  B: shared [K][ldb];  Wsl: 2 x KS x HP floats
template <int HD, int S, int NT>
__device__ __noinline__ void gemm_fwd_ws(const float* __restrict__ A, const float* __restrict__ Bm, int ldb, int K,
                                         const float* __restrict__ bias, float* __restrict__ P,
                                         float* __restrict__ Wsl) {
  using M = Map<HD, S, NT>;
  constexpr int HP = hp_of(HD), SP = M::SP, TM = M::TM, KS = 16, R4 = HP / 4;
  const M mp;
  const int m0 = mp.mt * TM, tid = threadIdx.x;
  float acc[TM][4];
#pragma unroll
  for (int j = 0; j < TM; ++j) {
    const float bb = bias[m0 + j];
    acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = bb;
  }
  const int nsl = (K + KS - 1) / KS;
  auto load = [&](int sl, int buf) {
    const int rows = min(KS, K - sl * KS);
    const float* src = A + (size_t)sl * KS * HP;
    float* dst = Wsl + buf * KS * HP;
    for (int idx = tid; idx < rows * R4; idx += NT) cp_async16(dst + 4 * idx, src + 4 * idx);
    cp_async_commit();
  };
  load(0, 0);
  for (int sl = 0; sl < nsl; ++sl) {
    if (sl + 1 < nsl) load(sl + 1, (sl + 1) & 1);
    else cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const int rows = min(KS, K - sl * KS);
    const float* ap = Wsl + (sl & 1) * KS * HP + m0;
    const float* bp = Bm + (size_t)sl * KS * ldb + mp.n0;
#pragma unroll 4
    for (int k = 0; k < rows; ++k) {
      const float4 b = *reinterpret_cast<const float4*>(bp + k * ldb);
      float a[TM];
#pragma unroll
      for (int q = 0; q < TM / 4; ++q) {
        const float4 av = *reinterpret_cast<const float4*>(ap + k * HP + 4 * q);
        a[4 * q] = av.x; a[4 * q + 1] = av.y; a[4 * q + 2] = av.z; a[4 * q + 3] = av.w;
      }
#pragma unroll
      for (int j = 0; j < TM; ++j) {
        acc[j][0] = fmaf(a[j], b.x, acc[j][0]); acc[j][1] = fmaf(a[j], b.y, acc[j][1]);
        acc[j][2] = fmaf(a[j], b.z, acc[j][2]); acc[j][3] = fmaf(a[j], b.w, acc[j][3]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < TM; ++j)
    *reinterpret_cast<float4*>(P + (m0 + j) * SP + mp.n0) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
}

// Column slices [rows][OS] of a global k-major tile [rows][HP] staged as [rows][OS + 4] (bank skew 20 -> conflict-free
// float4 reads by the four feature-threads of a warp).  Shared by the backward-delta and input-gradient GEMMs.
constexpr int OS = 16, OSP = OS + 4;
template <int NT>
__device__ __forceinline__ void load_col_slice(const float* __restrict__ A, int HP, int rows, int o0, float* dst) {
  for (int idx = threadIdx.x; idx < rows * (OS / 4); idx += NT) {
    const int r = idx / (OS / 4), c4 = idx - r * (OS / 4);
    cp_async16(dst + r * OSP + 4 * c4, A + (size_t)r * HP + o0 + 4 * c4);
  }
  cp_async_commit();
}

// D[i][n] <- D[i][n] * sum_o A[i][o] * Dl[o][n];  A: global [HID][HP];  Wsl: 2 x HID x OSP floats
template <int HD, int S, int NT>
__device__ __noinline__ void gemm_bwd_ws(const float* __restrict__ A, const float* __restrict__ Dl,
                                         float* __restrict__ D, float* __restrict__ Wsl) {
  using M = Map<HD, S, NT>;
  constexpr int HID = HD, HP = hp_of(HD), SP = M::SP, TM = M::TM, RS = 4 * M::WM;
  const M mp;
  float acc[TM][4];
#pragma unroll
  for (int j = 0; j < TM; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  constexpr int nsl = HID / OS;
  load_col_slice<NT>(A, HP, HID, 0, Wsl);
  for (int sl = 0; sl < nsl; ++sl) {
    if (sl + 1 < nsl) load_col_slice<NT>(A, HP, HID, (sl + 1) * OS, Wsl + ((sl + 1) & 1) * HID * OSP);
    else cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const float* ap = Wsl + (sl & 1) * HID * OSP + mp.mt * OSP;
    const float* bp = Dl + (size_t)sl * OS * SP + mp.n0;
#pragma unroll
    for (int o = 0; o < OS; o += 4) {
      float4 b[4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) b[kk] = *reinterpret_cast<const float4*>(bp + (o + kk) * SP);
#pragma unroll
      for (int j = 0; j < TM; ++j) {
        const float4 a = *reinterpret_cast<const float4*>(ap + j * RS * OSP + o);
        acc[j][0] = fmaf(a.x, b[0].x, acc[j][0]); acc[j][1] = fmaf(a.x, b[0].y, acc[j][1]);
        acc[j][2] = fmaf(a.x, b[0].z, acc[j][2]); acc[j][3] = fmaf(a.x, b[0].w, acc[j][3]);
        acc[j][0] = fmaf(a.y, b[1].x, acc[j][0]); acc[j][1] = fmaf(a.y, b[1].y, acc[j][1]);
        acc[j][2] = fmaf(a.y, b[1].z, acc[j][2]); acc[j][3] = fmaf(a.y, b[1].w, acc[j][3]);
        acc[j][0] = fmaf(a.z, b[2].x, acc[j][0]); acc[j][1] = fmaf(a.z, b[2].y, acc[j][1]);
        acc[j][2] = fmaf(a.z, b[2].z, acc[j][2]); acc[j][3] = fmaf(a.z, b[2].w, acc[j][3]);
        acc[j][0] = fmaf(a.w, b[3].x, acc[j][0]); acc[j][1] = fmaf(a.w, b[3].y, acc[j][1]);
        acc[j][2] = fmaf(a.w, b[3].z, acc[j][2]); acc[j][3] = fmaf(a.w, b[3].w, acc[j][3]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < TM; ++j) {
    float* dp = D + (mp.mt + j * RS) * SP + mp.n0;
    float4 d = *reinterpret_cast<const float4*>(dp);
    d.x *= acc[j][0]; d.y *= acc[j][1]; d.z *= acc[j][2]; d.w *= acc[j][3];
    *reinterpret_cast<float4*>(dp) = d;
  }
}

// Xb[i][s] = sum_o W1k[i][o] * Dl[o][s], i < M;  W1k: global [in][HP];  Wsl: 2 x rows8 x OSP floats
template <int HD, int S, int NT>
__device__ __noinline__ void gemm_dx_ws(const float* __restrict__ W1k, const float* __restrict__ Dl, int M,
                                        float* __restrict__ Xb, int ldx, float* __restrict__ Wsl) {
  constexpr int SP = S + 4, NTN = S / 4, MG = NT / NTN, JM = 8, HID = HD, HP = hp_of(HD);
  const int tid = threadIdx.x, nt = tid % NTN, mg = tid / NTN;
  const int J = max(0, (M - mg + MG - 1) / MG);
  const int rows = (M + 3) & ~3;       // <= in rows of the blob (pad rows are zero there)
  float acc[JM][4];
#pragma unroll
  for (int j = 0; j < JM; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  constexpr int nsl = HID / OS;
  const int stride = ((rows + 7) & ~7) * OSP;
  load_col_slice<NT>(W1k, HP, M, 0, Wsl);
  for (int sl = 0; sl < nsl; ++sl) {
    if (sl + 1 < nsl) load_col_slice<NT>(W1k, HP, M, (sl + 1) * OS, Wsl + ((sl + 1) & 1) * stride);
    else cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const float* wp = Wsl + (sl & 1) * stride;
    const float* dp = Dl + (size_t)sl * OS * SP + 4 * nt;
#pragma unroll
    for (int o = 0; o < OS; o += 4) {
      float4 d[4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) d[kk] = *reinterpret_cast<const float4*>(dp + (o + kk) * SP);
#pragma unroll
      for (int j = 0; j < JM; ++j)
        if (j < J) {
          const float4 w = *reinterpret_cast<const float4*>(wp + (mg + MG * j) * OSP + o);
          acc[j][0] = fmaf(w.x, d[0].x, acc[j][0]); acc[j][1] = fmaf(w.x, d[0].y, acc[j][1]);
          acc[j][2] = fmaf(w.x, d[0].z, acc[j][2]); acc[j][3] = fmaf(w.x, d[0].w, acc[j][3]);
          acc[j][0] = fmaf(w.y, d[1].x, acc[j][0]); acc[j][1] = fmaf(w.y, d[1].y, acc[j][1]);
          acc[j][2] = fmaf(w.y, d[1].z, acc[j][2]); acc[j][3] = fmaf(w.y, d[1].w, acc[j][3]);
          acc[j][0] = fmaf(w.z, d[2].x, acc[j][0]); acc[j][1] = fmaf(w.z, d[2].y, acc[j][1]);
          acc[j][2] = fmaf(w.z, d[2].z, acc[j][2]); acc[j][3] = fmaf(w.z, d[2].w, acc[j][3]);
          acc[j][0] = fmaf(w.w, d[3].x, acc[j][0]); acc[j][1] = fmaf(w.w, d[3].y, acc[j][1]);
          acc[j][2] = fmaf(w.w, d[3].z, acc[j][2]); acc[j][3] = fmaf(w.w, d[3].w, acc[j][3]);
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < JM; ++j)
    if (j < J)
      *reinterpret_cast<float4*>(Xb + (mg + MG * j) * ldx + 4 * nt) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
}

// Copy rows [0, nrows) x S columns of the global observation tile (row stride ldx) into shared memory [nrows][S + 4]
template <int S, int NT>
__device__ __forceinline__ void stage_x_tile(const float* __restrict__ Xg, int ldx, int nrows, float* __restrict__ Xs) {
  constexpr int SP = S + 4, C4 = S / 4;
  for (int idx = threadIdx.x; idx < nrows * C4; idx += NT) {
    const int r = idx / C4, c4 = idx - r * C4;
    cp_async16(Xs + r * SP + 4 * c4, Xg + (size_t)r * ldx + 4 * c4);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
}

// Shared-memory views of one CTA.  X and Z hold one column per THREAD (row stride XS = NT + 4); the
// activation tiles H1/D1/H2/D2 hold one S-sample sub-tile (row stride SP = S + 4) and are reused by the
// NT/S sub-tiles of a chunk.  X/Z pointers passed to the mlp_* helpers are already offset to the sub-tile.
struct Tiles {
  float *W, *dW, *X, *H1, *D1, *H2, *D2, *Z;
  float* R;   // wide nets: shared staging region (observation sub-tile + double-buffered weight slices)
};

// X -> H1 -> H2 (-> Zout rows a and 4 + a: consumers add the two).  FULL: also store activation derivatives.
// HD == 64 (tensor-core path): every step is local to the 16-sample stripe owned by one warp pair, so only the
// pair's 64-thread named barrier is used and the pairs of a CTA run asynchronously.  HD == 256 (FFMA path):
// CTA-wide tiles and barriers.  Ends with a barrier of the respective scope.
template <int HD, int S, int NT, bool FULL, bool OUT>
__device__ __forceinline__ void mlp_forward(const NetL& L, const Tiles& t, float* Zout) {
  constexpr int XS = NT + 4, HID = HD;
  if constexpr (HD == 64) {
    gemm_fwd_mma<S, NT, hp_of(HD)>(t.W + L.o_w1, t.W + L.o_w1l, t.X, XS, L.in8, t.W + L.o_b1, t.H1, false);
    act_pass_frag<S, NT>(t.H1, FULL ? t.D1 : nullptr, L.hact, nullptr, nullptr, 0, nullptr, 0);
    pair_sync();
    gemm_fwd_mma<S, NT, hp_of(HD)>(t.W + L.o_w2, t.W + L.o_w2l, t.H1, S + 4, HID, t.W + L.o_b2, t.H2, true);
    act_pass_frag<S, NT>(t.H2, FULL ? t.D2 : nullptr, L.hact, OUT ? t.W + L.o_w3 : nullptr, t.W + L.o_b3, L.out,
                         Zout, XS);
    pair_sync();
  } else {
    // R = [ observation sub-tile  Xs: inp x (S+4) | weight slices ]
    float* Xs = t.R;
    float* Wsl = t.R + L.inp * (S + 4);
    stage_x_tile<S, NT>(t.X, XS, L.in, Xs);
    gemm_fwd_ws<HD, S, NT>(t.W + L.o_w1, Xs, S + 4, L.in, t.W + L.o_b1, t.H1, Wsl);
    act_pass<HD, S, NT>(t.H1, FULL ? t.D1 : nullptr, L.hact);
    __syncthreads();
    gemm_fwd_ws<HD, S, NT>(t.W + L.o_w2, t.H1, S + 4, HID, t.W + L.o_b2, t.H2, Wsl);
    act_pass<HD, S, NT>(t.H2, FULL ? t.D2 : nullptr, L.hact);
    __syncthreads();
    if (OUT) {
      out_layer<HD, S, NT>(t.W + L.o_w3, t.W + L.o_b3, t.H2, L.out, Zout, XS);
      __syncthreads();
    }
  }
}

// Given Zbar in t.Z (rows 0..out-1): accumulate weight grads into t.dW (torch flat layout) if WANT_DW and
// write the observation gradient into rows [0, L.obs) of t.X if want_dx.  Requires a FULL forward of the
// same sub-tile.  HD == 64: delta2 / delta1 / dX are stripe-local (pair barriers); only the weight-gradient
// reductions over samples are bracketed by CTA barriers, with the small jobs dealt to different warps.
template <int HD, int S, int NT, bool WANT_DW>
__device__ __forceinline__ void mlp_backward(const NetL& L, const Tiles& t, bool want_dx) {
  constexpr int XS = NT + 4, SP = S + 4, HID = HD;
  if constexpr (HD == 64) {
    constexpr int HPc = hp_of(HD);
    if (WANT_DW) {   // delta2 overwrites D2 in place: dW3 needs H2 only, db3 needs Zbar only -> do them in the dW phase
    }
    delta_from_out_frag<S, NT>(t.W + L.o_w3, t.Z, XS, L.out, t.D2);               // D2 <- delta2 (stripe)
    pair_sync();
    gemm_bwd_mma<S, NT, HPc>(t.W + L.o_w2, t.W + L.o_w2l, t.D2, t.D1);            // D1 <- delta1 (stripe)
    if (WANT_DW) {
      __syncthreads();                                                            // every stripe's deltas are ready
      dw_accum_mma<S, NT>(t.D2, SP, t.H1, SP, HID, t.dW + L.d_w2, L.ldw2, 0, true);
      dw_accum_mma<S, NT>(t.D1, SP, t.X, XS, L.in, t.dW + L.d_w1, L.in, NT / 64, false);
      rowsum_accum<HD, S, NT>(t.D2, SP, HID, t.dW + L.d_b2, NT / 4);
      rowsum_accum<HD, S, NT>(t.D1, SP, HID, t.dW + L.d_b1, NT / 4 + 64);
      dw_accum<HD, S, NT, 1, 4>(t.Z, XS, L.out, t.H2, SP, HID, t.dW + L.d_w3, HID, 3 * NT / 4, true);
      rowsum_accum<HD, S, NT>(t.Z, XS, L.out, t.dW + L.d_b3, 3 * NT / 4 + 32);
      __syncthreads();                                                            // X / tiles may be overwritten
    } else {
      pair_sync();
    }
    if (want_dx) {
      gemm_dx_mma<S, NT, HPc>(t.W + L.o_w1, t.W + L.o_w1l, t.D1, L.obs, t.X, XS);
      pair_sync();
    }
  } else {
    if (WANT_DW) {
      dw_accum<HD, S, NT, 1, 4>(t.Z, XS, L.out, t.H2, SP, HID, t.dW + L.g_w3, HID);
      rowsum_accum<HD, S, NT>(t.Z, XS, L.out, t.dW + L.g_b3);
    }
    delta_from_out<HD, S, NT>(t.W + L.o_w3, t.Z, XS, L.out, t.D2);  // D2 <- delta2
    __syncthreads();
    gemm_bwd_ws<HD, S, NT>(t.W + L.o_w2, t.D2, t.D1, t.R);          // D1 <- delta1 (weight slices through R)
    if (WANT_DW) {
      dw_accum<HD, S, NT, 4, 4>(t.D2, SP, HID, t.H1, SP, HID, t.dW + L.g_w2, HID);
      rowsum_accum<HD, S, NT>(t.D2, SP, HID, t.dW + L.g_b2);
    }
    __syncthreads();
    if (WANT_DW) {
      stage_x_tile<S, NT>(t.X, XS, L.in, t.R);                      // observation sub-tile back into shared memory
      dw_accum<HD, S, NT, 4, 4>(t.D1, SP, HID, t.R, SP, L.in, t.dW + L.g_w1, L.in);
      rowsum_accum<HD, S, NT>(t.D1, SP, HID, t.dW + L.g_b1);
      __syncthreads();
    }
    if (want_dx) gemm_dx_ws<HD, S, NT>(t.W + L.o_w1, t.D1, L.obs, t.X, XS, t.R);
    __syncthreads();
  }
}

}  // namespace gops
