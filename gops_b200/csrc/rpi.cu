// RPI (relaxed policy iteration, reference gops/algorithm/rpi.py) on pyth_oscillatorconti with a StateValue MLP
// [2 -> 64 -> 64 -> 1].  Three entry points share the tile functions below:
//   gops_b200_rpi_policy       greedy action and worst disturbance from the target value's input gradient (any batch)
//   gops_b200_rpi_loss_grad    one Hamiltonian loss mean|c + dV/dx . f| and its parameter gradient
//   gops_b200_rpi_newton       one Newton iteration (RPI.local_update) in ONE launch: the whole policy-evaluation loop,
//                              its stopping test and the target copy run on the device
//
// A tile is 64 samples on a CTA of 256 threads.  Thread t owns rows rg + 16 r and columns cg + 16 c (r, c < 4) of every
// [64 x 64] plane, rg = t / 16, cg = t % 16; the 16 lanes of one row group reduce per-sample sums with shuffles.
// Planes and the W2 block of a parameter set live in shared memory with a row stride of 65 floats, so that row- and
// column-wise reads of both GEMM directions are free of bank conflicts.  All arithmetic is fp32 on the CUDA cores
// (every product is one correctly rounded fma), and every reduction runs in a fixed order.
//
// dV/dx . f is the forward-mode tangent of V along f (DESIGN.md, "RPI"):
//   z1 = W1 x + b1, h1 = s(z1), z1' = W1 f, h1' = s'(z1) z1',  z2 = W2 h1 + b2, z2' = W2 h1', h2' = s'(z2) z2',
//   V' = W3 h2'.   With q = sign(c + V') / B the reverse sweep is
//   dW3 = q h2',  gz2' = q W3 s'(z2),  gz2 = q W3 z2' s''(z2),  dW2 = gz2' h1'^T + gz2 h1^T,  db2 = gz2,
//   gh1' = W2^T gz2',  gh1 = W2^T gz2,  gz1' = gh1' s'(z1),  gz1 = gh1 s'(z1) + gh1' z1' s''(z1),
//   dW1 = gz1' f^T + gz1 x^T,  db1 = gz1,  db3 = 0.
#include "gops_b200.h"

#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math.h>

#include <string>

#include "adam_math.cuh"
#include "host_util.h"
#include "models.cuh"

namespace cg = cooperative_groups;
using gops::DevGuard;
using gops::fail;
using gops::g_launches;

namespace {

constexpr int NT = 256;            // threads per tile
constexpr int TS = 64;             // samples per tile
constexpr int HID = 64;
constexpr int LD = 65;             // padded row stride of planes and of W2
constexpr int NPARAM = 2 * HID + HID + HID * HID + HID + HID + 1;   // 4417, torch parameters() order
constexpr int O_B1 = 2 * HID, O_W2 = 3 * HID, O_B2F = O_W2 + HID * HID, O_W3F = O_B2F + HID, O_B3F = O_W3F + HID;
constexpr int O_B2 = O_W2 + HID * LD, O_W3 = O_B2 + HID, O_B3 = O_W3 + HID;   // padded shared-memory layout
constexpr int SPARAM = O_B3 + 1;   // 4481
constexpr int PLANE = TS * LD;
constexpr int NPL = 8;
constexpr int PER_T = (NPARAM + NT - 1) / NT;   // flat parameters owned by one thread for Adam (18)
constexpr int MAX_CLUSTER = 8;

__device__ __forceinline__ int smem_index(int i) {
  if (i < O_W2) return i;
  if (i < O_B2F) { const int r = i - O_W2; return O_W2 + (r / HID) * LD + (r % HID); }
  return i + (O_B2 - O_B2F);
}

struct Consts {
  float act_low[2], act_high[2];   // model bounds of [u, w]: [-5, 5], [-1/gamma_atte, 1/gamma_atte]
  float th[2];                     // state_threshold
  float dt;                        // 1/200
  float k3;                        // float(1 / (2 gamma_atte^2))
  float gam2;                      // float(gamma_atte^2)
  float wcoef;                     // float(0.5 / gamma_atte^2), worst_adv
  float inv_B;
};

// shared-memory carve (floats): P, T, G, 8 planes, per-sample arrays
struct Smem {
  float* P; float* T; float* G; float* pl[NPL];
  float* x;   // [64][2] current states of the tile
  float* xn;  // [64][2] next states
  float* sx;  // [64][2] set_state
  float* sa;  // [64][2] raw (a, w) of the target policy at set_state
  float* a;   // [64][2] raw (a, w) at x
  float* f;   // [64][2] delta_state of the wrapped forward
  float* c;   // [64] cost
  float* absh;  // [64]
  float* red;   // [4]: 0 loss partial, 1 |H| partial, 2 H_before partial
};
constexpr int SMEM_FLOATS = 2 * SPARAM + NPARAM + NPL * PLANE + 6 * 2 * TS + 2 * TS + 4;

__device__ __forceinline__ Smem carve(float* s) {
  Smem m;
  m.P = s; s += SPARAM;
  m.T = s; s += SPARAM;
  m.G = s; s += NPARAM;
  for (int i = 0; i < NPL; ++i) { m.pl[i] = s; s += PLANE; }
  m.x = s; s += 2 * TS;
  m.xn = s; s += 2 * TS;
  m.sx = s; s += 2 * TS;
  m.sa = s; s += 2 * TS;
  m.a = s; s += 2 * TS;
  m.f = s; s += 2 * TS;
  m.c = s; s += TS;
  m.absh = s; s += TS;
  m.red = s;
  return m;
}

__device__ void load_params(float* dst, const float* __restrict__ src) {
  for (int i = threadIdx.x; i < NPARAM; i += NT) dst[smem_index(i)] = src[i];
}

// sigma''(z) from z, h = sigma(z), d = sigma'(z)
template <int ACT>
__device__ __forceinline__ float act_dd(float z, float h, float d) {
  if constexpr (ACT == GOPS_ACT_ELU || ACT == GOPS_ACT_SELU) return z > 0.f ? 0.f : d;
  else if constexpr (ACT == GOPS_ACT_GELU) return 0.39894228040143267794f * expf(-0.5f * z * z) * (2.f - z * z);
  else if constexpr (ACT == GOPS_ACT_SIGMOID) return d * (1.f - 2.f * h);
  else if constexpr (ACT == GOPS_ACT_TANH) return -2.f * h * d;
  else return 0.f;   // relu, linear
}

// 16-lane (one row group) sum, fixed butterfly order: every lane gets the same value
__device__ __forceinline__ float row_sum(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Layer 1 on planes: pl[0] = h1, pl[1] = d1; with TAN pl[2] = z1' (tangent f), pl[3] = h1' = d1 z1', pl[4] = s''(z1).
template <int ACT, bool TAN>
__device__ void layer1(const float* W, const float* x, const float* f, float* const* pl) {
  const int rg = threadIdx.x >> 4, cg = threadIdx.x & 15;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int s = rg + 16 * r;
    const float x0 = x[2 * s], x1 = x[2 * s + 1];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int k = cg + 16 * c;
      const float z = fmaf(W[2 * k + 1], x1, fmaf(W[2 * k], x0, W[O_B1 + k]));
      float h, d;
      gops::act_fwd_grad_t<ACT>(z, h, d);
      pl[0][s * LD + k] = h;
      pl[1][s * LD + k] = d;
      if constexpr (TAN) {
        const float zt = fmaf(W[2 * k + 1], f[2 * s + 1], __fmul_rn(W[2 * k], f[2 * s]));
        pl[2][s * LD + k] = zt;
        pl[3][s * LD + k] = __fmul_rn(d, zt);
        pl[4][s * LD + k] = act_dd<ACT>(z, h, d);
      }
    }
  }
}

// acc[r][c] (+)= sum_k A[row r][k] W2[col c][k]  (forward layer 2, both operands read along k)
template <bool DUAL>
__device__ __forceinline__ void gemm_fwd(const float* W, const float* A, const float* Ad, float (&acc)[4][4],
                                         float (&accd)[4][4]) {
  const int rg = threadIdx.x >> 4, cg = threadIdx.x & 15;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float b = W[O_B2 + cg + 16 * c];
#pragma unroll
    for (int r = 0; r < 4; ++r) { acc[r][c] = b; accd[r][c] = 0.f; }
  }
#pragma unroll 4
  for (int k = 0; k < HID; ++k) {
    float a[4], ad[4], w[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      a[r] = A[(rg + 16 * r) * LD + k];
      if constexpr (DUAL) ad[r] = Ad[(rg + 16 * r) * LD + k];
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) w[c] = W[O_W2 + (cg + 16 * c) * LD + k];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        acc[r][c] = fmaf(a[r], w[c], acc[r][c]);
        if constexpr (DUAL) accd[r][c] = fmaf(ad[r], w[c], accd[r][c]);
      }
  }
}

// acc[r][c] = sum_j A[row r][j] W2[j][col c]  (backward through layer 2)
template <bool DUAL>
__device__ __forceinline__ void gemm_bwd(const float* W, const float* A, const float* Ad, float (&acc)[4][4],
                                         float (&accd)[4][4]) {
  const int rg = threadIdx.x >> 4, cg = threadIdx.x & 15;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) { acc[r][c] = 0.f; accd[r][c] = 0.f; }
#pragma unroll 4
  for (int j = 0; j < HID; ++j) {
    float a[4], ad[4], w[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      a[r] = A[(rg + 16 * r) * LD + j];
      if constexpr (DUAL) ad[r] = Ad[(rg + 16 * r) * LD + j];
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) w[c] = W[O_W2 + j * LD + cg + 16 * c];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        acc[r][c] = fmaf(a[r], w[c], acc[r][c]);
        if constexpr (DUAL) accd[r][c] = fmaf(ad[r], w[c], accd[r][c]);
      }
  }
}

// Greedy action and worst disturbance at x with the value net W (ApproxContainer.action_and_adversary):
// p = dV/dx, a = -0.5 x0 p1 (best_act), w = float(0.5/gamma^2) x1 p1 (worst_adv).  out: [64][2] raw (a, w).
template <int ACT>
__device__ void policy_tile(const Smem& m, const float* W, const float* x, float* out, const Consts& k) {
  float* const* pl = m.pl;
  layer1<ACT, false>(W, x, nullptr, pl);
  __syncthreads();
  const int rg = threadIdx.x >> 4, cg = threadIdx.x & 15;
  float acc[4][4], accd[4][4];
  gemm_fwd<false>(W, pl[0], nullptr, acc, accd);
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = cg + 16 * c;
      float h, d;
      gops::act_fwd_grad_t<ACT>(acc[r][c], h, d);
      pl[2][(rg + 16 * r) * LD + j] = __fmul_rn(W[O_W3 + j], d);   // dV/dz2
    }
  __syncthreads();
  gemm_bwd<false>(W, pl[2], nullptr, acc, accd);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int s = rg + 16 * r;
    float p0 = 0.f, p1 = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int kk = cg + 16 * c;
      const float g1 = __fmul_rn(acc[r][c], pl[1][s * LD + kk]);
      p0 = fmaf(W[2 * kk], g1, p0);
      p1 = fmaf(W[2 * kk + 1], g1, p1);
    }
    p0 = row_sum(p0);
    p1 = row_sum(p1);
    (void)p0;   // g(x) = [0, x0], k(x) = [0, x1]: only dV/dx1 enters
    if (cg == 0) {
      out[2 * s] = __fmul_rn(-0.5f, __fmul_rn(x[2 * s], p1));
      out[2 * s + 1] = __fmul_rn(k.wcoef, __fmul_rn(x[2 * s + 1], p1));
    }
  }
  __syncthreads();
}

__device__ __forceinline__ gops::KParams wrap_params(const Consts& k) {
  gops::KParams p;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    p.min_action[j] = -1.f; p.max_action[j] = 1.f;
    p.act_low[j] = k.act_low[j]; p.act_high[j] = k.act_high[j];
  }
  return p;
}

// delta_state f(x, u, w) and cost c of pyth_oscillatorconti (model.forward), fp32 in the reference's operation order
__device__ __forceinline__ void osc_f(const Consts& k, float x0, float x1, float u, float w, float& f0, float& f1) {
  f0 = __fmul_rn(-0.25f, x0);
  float t = __fmul_rn(0.5f, __fmul_rn(__fmul_rn(x0, x0), x1));
  t = __fsub_rn(t, __fmul_rn(k.k3, __fmul_rn(__fmul_rn(x1, x1), x1)));
  t = __fsub_rn(t, __fmul_rn(0.5f, x1));
  t = __fadd_rn(t, __fmul_rn(x0, u));
  f1 = __fadd_rn(t, __fmul_rn(x1, w));
}

// (x, raw a/w) -> f and c of the WRAPPED forward (ScaleAction -> ClipAction -> model): threads < 64
__device__ void prep_wrapped(const Smem& m, const float* x, const float* raw, const Consts& k) {
  const int s = threadIdx.x;
  if (s < TS) {
    const gops::KParams p = wrap_params(k);
    float gg = 1.f;
    const float u = gops::wrap_action<gops::WrapFixed<gops::kWrapActionScale | gops::kWrapClipAction>>(p, 0, raw[2 * s], gg);
    const float w = gops::wrap_action<gops::WrapFixed<gops::kWrapActionScale | gops::kWrapClipAction>>(p, 1, raw[2 * s + 1], gg);
    const float x0 = x[2 * s], x1 = x[2 * s + 1];
    osc_f(k, x0, x1, u, w, m.f[2 * s], m.f[2 * s + 1]);
    float c = __fadd_rn(__fmul_rn(x0, x0), __fmul_rn(x1, x1));
    c = __fadd_rn(c, __fmul_rn(u, u));
    m.c[s] = __fsub_rn(c, __fmul_rn(k.gam2, __fmul_rn(w, w)));
  }
  __syncthreads();
}

// Hamiltonian H_s = c_s + V'_s at x (f, c prepared); returns in m.absh[s] = |H_s|.  GRAD: the reverse sweep writes the
// tile's gradient of sum_s |H_s| inv_B into m.G (flat order).
template <int ACT, bool GRAD>
__device__ void hamiltonian_tile(const Smem& m, const float* W, const float* x, const Consts& k) {
  float* const* pl = m.pl;
  layer1<ACT, true>(W, x, m.f, pl);
  __syncthreads();
  const int rg = threadIdx.x >> 4, cg = threadIdx.x & 15;
  float acc[4][4], accd[4][4];
  gemm_fwd<true>(W, pl[0], pl[3], acc, accd);      // z2, z2'
  float hd2[4][4], a2[4][4], b2[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    float vd = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = cg + 16 * c;
      float h, d;
      gops::act_fwd_grad_t<ACT>(acc[r][c], h, d);
      hd2[r][c] = __fmul_rn(d, accd[r][c]);
      vd = fmaf(W[O_W3 + j], hd2[r][c], vd);
      if constexpr (GRAD) {
        a2[r][c] = __fmul_rn(W[O_W3 + j], d);
        b2[r][c] = __fmul_rn(__fmul_rn(W[O_W3 + j], accd[r][c]), act_dd<ACT>(acc[r][c], h, d));
      }
    }
    vd = row_sum(vd);
    const int s = rg + 16 * r;
    const float H = __fadd_rn(m.c[s], vd);
    if (cg == 0) m.absh[s] = fabsf(H);
    if constexpr (GRAD) {
      const float q = H > 0.f ? k.inv_B : (H < 0.f ? -k.inv_B : 0.f);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = cg + 16 * c;
        pl[5][s * LD + j] = __fmul_rn(q, a2[r][c]);     // gz2'
        pl[6][s * LD + j] = __fmul_rn(q, b2[r][c]);     // gz2
        pl[7][s * LD + j] = __fmul_rn(q, hd2[r][c]);    // dW3 terms
      }
    }
  }
  __syncthreads();
  if constexpr (GRAD) {
    gemm_bwd<true>(W, pl[5], pl[6], acc, accd);    // acc = gh1', accd = gh1
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int o = (rg + 16 * r) * LD + cg + 16 * c;
        const float d1 = pl[1][o], zt = pl[2][o], s1 = pl[4][o];
        const float gzt = __fmul_rn(acc[r][c], d1);
        const float gz = fmaf(__fmul_rn(acc[r][c], zt), s1, __fmul_rn(accd[r][c], d1));
        pl[2][o] = gzt;    // gz1'  (owner-only element: z1' is read here last)
        pl[4][o] = gz;     // gz1
      }
    __syncthreads();
    // dW2[j][kk] = sum_s gz2'[s][j] h1'[s][kk] + gz2[s][j] h1[s][kk]
    float g[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) g[a][c] = 0.f;
#pragma unroll 2
    for (int s = 0; s < TS; ++s) {
      float ga[4], gb[4], hd[4], h[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) { ga[a] = pl[5][s * LD + rg + 16 * a]; gb[a] = pl[6][s * LD + rg + 16 * a]; }
#pragma unroll
      for (int c = 0; c < 4; ++c) { hd[c] = pl[3][s * LD + cg + 16 * c]; h[c] = pl[0][s * LD + cg + 16 * c]; }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) g[a][c] = fmaf(gb[a], h[c], fmaf(ga[a], hd[c], g[a][c]));
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) m.G[O_W2 + (rg + 16 * a) * HID + cg + 16 * c] = g[a][c];
    // dW1 [64][2], db1, db2, dW3, db3
    for (int o = threadIdx.x; o < 5 * HID + 1; o += NT) {
      float sum = 0.f;
      if (o < 2 * HID) {
        const int kk = o >> 1, mm = o & 1;
        for (int s = 0; s < TS; ++s)
          sum = fmaf(pl[4][s * LD + kk], x[2 * s + mm], fmaf(pl[2][s * LD + kk], m.f[2 * s + mm], sum));
        m.G[o] = sum;
      } else if (o < 3 * HID) {
        const int kk = o - 2 * HID;
        for (int s = 0; s < TS; ++s) sum = __fadd_rn(sum, pl[4][s * LD + kk]);
        m.G[O_B1 + kk] = sum;
      } else if (o < 4 * HID) {
        const int j = o - 3 * HID;
        for (int s = 0; s < TS; ++s) sum = __fadd_rn(sum, pl[6][s * LD + j]);
        m.G[O_B2F + j] = sum;
      } else if (o < 5 * HID) {
        const int j = o - 4 * HID;
        for (int s = 0; s < TS; ++s) sum = __fadd_rn(sum, pl[7][s * LD + j]);
        m.G[O_W3F + j] = sum;
      } else {
        m.G[O_B3F] = 0.f;
      }
    }
    __syncthreads();
  }
}

// sum_s |H_s| of the tile in sample order (thread 0)
__device__ __forceinline__ float tile_abs_sum(const Smem& m) {
  float s = 0.f;
  for (int i = 0; i < TS; ++i) s = __fadd_rn(s, m.absh[i]);
  return s;
}

// ------------------------------------------------------------------------------------------------------------------
template <int ACT>
__global__ void __launch_bounds__(NT, 1) rpi_policy_kernel(const float* __restrict__ params, const float* __restrict__ obs,
                                                           long long B, Consts k, float* __restrict__ out) {
  extern __shared__ float smem[];
  const Smem m = carve(smem);
  load_params(m.T, params);
  const long long base = (long long)blockIdx.x * TS;
  for (int i = threadIdx.x; i < 2 * TS; i += NT) {
    const long long g = base * 2 + i;
    m.x[i] = g < 2 * B ? obs[g] : 0.f;
  }
  __syncthreads();
  policy_tile<ACT>(m, m.T, m.x, m.a, k);
  for (int i = threadIdx.x; i < 2 * TS; i += NT) {
    const long long g = base * 2 + i;
    if (g < 2 * B) out[g] = m.a[i];
  }
}

// One tile of the single-step Hamiltonian loss: partial gradient [NPARAM] and partial sum_s |H_s| per tile.
template <int ACT>
__global__ void __launch_bounds__(NT, 1) rpi_loss_tile_kernel(const float* __restrict__ params, const float* __restrict__ obs,
                                                              const float* __restrict__ act, Consts k,
                                                              float* __restrict__ part_g, float* __restrict__ part_l) {
  extern __shared__ float smem[];
  const Smem m = carve(smem);
  load_params(m.P, params);
  const long long base = (long long)blockIdx.x * TS * 2;
  for (int i = threadIdx.x; i < 2 * TS; i += NT) { m.x[i] = obs[base + i]; m.a[i] = act[base + i]; }
  __syncthreads();
  prep_wrapped(m, m.x, m.a, k);
  hamiltonian_tile<ACT, true>(m, m.P, m.x, k);
  for (int i = threadIdx.x; i < NPARAM; i += NT) part_g[(long long)blockIdx.x * NPARAM + i] = m.G[i];
  if (threadIdx.x == 0) part_l[blockIdx.x] = tile_abs_sum(m);
}

// Tile partials -> gradient and loss, summed over tiles in tile order (the order of the Newton kernel's cluster sum).
__global__ void rpi_reduce_kernel(const float* __restrict__ part_g, const float* __restrict__ part_l, int tiles, float inv_B,
                                  float* __restrict__ grad, float* __restrict__ loss) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < NPARAM) {
    float g = part_g[i];
    for (int r = 1; r < tiles; ++r) g = __fadd_rn(g, part_g[(long long)r * NPARAM + i]);
    grad[i] = g;
  }
  if (i == 0) {
    float l = part_l[0];
    for (int r = 1; r < tiles; ++r) l = __fadd_rn(l, part_l[r]);
    *loss = __fmul_rn(l, inv_B);
  }
}

struct NewtonArgs {
  float* params; float* target; float* exp_avg; float* exp_avg_sq;
  float* state;            // [B][2] sampler states, updated
  const int* max_step;     // [B] max_step_per_episode
  int* counter;            // [1] the model's step_per_episode (one value for every sample), updated
  const float* draws;      // [rows][B][2] reset() draws: row 0 set_state, row n the draw of inner step n
  int rows, max_steps;
  long long step0;         // Adam steps taken before this launch
  double lr, beta1, beta2, eps;
  float* out;              // [8]: n, last loss, H_before, H_after, draws exhausted
  float* trace;            // [max_steps][2] (loss, H_after) per inner step, or NULL
  long long B;
};

// sum over the cluster's CTAs of a shared-memory scalar, in rank order
__device__ __forceinline__ float cluster_sum(cg::cluster_group& cl, float* slot, int nc) {
  float s = *cl.map_shared_rank(slot, 0);
  for (int r = 1; r < nc; ++r) s = __fadd_rn(s, *cl.map_shared_rank(slot, r));
  return s;
}

template <int ACT>
__global__ void __launch_bounds__(NT, 1) rpi_newton_kernel(NewtonArgs A, Consts k) {
  extern __shared__ float smem[];
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank(), nc = (int)cl.num_blocks();
  const Smem m = carve(smem);
  const long long base = (long long)rank * TS;
  const int tid = threadIdx.x;
  load_params(m.P, A.params);
  load_params(m.T, A.target);
  float mom[PER_T], vel[PER_T];
#pragma unroll
  for (int q = 0; q < PER_T; ++q) {
    const int i = tid + q * NT;
    mom[q] = i < NPARAM ? A.exp_avg[i] : 0.f;
    vel[q] = i < NPARAM ? A.exp_avg_sq[i] : 0.f;
  }
  int maxst = 0;
  if (tid < TS) maxst = A.max_step[base + tid];
  int cnt = *A.counter;
  for (int i = tid; i < 2 * TS; i += NT) {
    m.x[i] = A.state[base * 2 + i];
    m.sx[i] = A.draws[base * 2 + i];
  }
  __syncthreads();
  // set_state: actions of the target net (constant for the iteration), H_before with the current net
  policy_tile<ACT>(m, m.T, m.sx, m.sa, k);
  prep_wrapped(m, m.sx, m.sa, k);
  hamiltonian_tile<ACT, false>(m, m.P, m.sx, k);
  if (tid == 0) m.red[2] = tile_abs_sum(m);
  cl.sync();
  const float h_before = __fmul_rn(cluster_sum(cl, m.red + 2, nc), k.inv_B);
  const float omb1 = (float)(1.0 - A.beta1), b2f = (float)A.beta2, omb2 = (float)(1.0 - A.beta2), epsf = (float)A.eps;
  int n = 0;
  float loss = 0.f, h_after = 0.f;
  bool exhausted = false;
  while (true) {
    ++n;
    // RPI.sample: target policy at x, raw Euler step of the unwrapped model, done / truncation, reset draws
    policy_tile<ACT>(m, m.T, m.x, m.a, k);
    if (tid < TS) {
      const int s = tid;
      const float x0 = m.x[2 * s], x1 = m.x[2 * s + 1];
      float f0, f1;
      osc_f(k, x0, x1, m.a[2 * s], m.a[2 * s + 1], f0, f1);
      const float n0 = __fadd_rn(x0, __fmul_rn(f0, k.dt)), n1 = __fadd_rn(x1, __fmul_rn(f1, k.dt));
      const bool done = fabsf(n0) > k.th[0] || fabsf(n1) > k.th[1];
      const bool trunc = cnt + 1 > maxst;
      const float* d = A.draws + ((long long)n * A.B + base + s) * 2;
      m.xn[2 * s] = (done || trunc) ? d[0] : n0;
      m.xn[2 * s + 1] = (done || trunc) ? d[1] : n1;
    }
    ++cnt;
    prep_wrapped(m, m.x, m.a, k);
    hamiltonian_tile<ACT, true>(m, m.P, m.x, k);
    if (tid == 0) m.red[0] = tile_abs_sum(m);
    cl.sync();
    loss = __fmul_rn(cluster_sum(cl, m.red, nc), k.inv_B);
    {
      const long long st = A.step0 + n;
      const double bc1 = 1.0 - pow(A.beta1, (double)st), bc2 = 1.0 - pow(A.beta2, (double)st);
      const float step_size = (float)(A.lr / bc1), bc2_sqrt = (float)sqrt(bc2);
#pragma unroll
      for (int q = 0; q < PER_T; ++q) {
        const int i = tid + q * NT;
        if (i < NPARAM) {
          float g = *cl.map_shared_rank(m.G + i, 0);
          for (int r = 1; r < nc; ++r) g = __fadd_rn(g, *cl.map_shared_rank(m.G + i, r));
          gops::adam_update(g, m.P[smem_index(i)], mom[q], vel[q], omb1, b2f, omb2, epsf, step_size, bc2_sqrt);
        }
      }
    }
    for (int i = tid; i < 2 * TS; i += NT) m.x[i] = m.xn[i];
    __syncthreads();
    // stopping test: H on set_state with the updated net (f and c of set_state again: the loss overwrote them)
    prep_wrapped(m, m.sx, m.sa, k);
    hamiltonian_tile<ACT, false>(m, m.P, m.sx, k);
    if (tid == 0) m.red[1] = tile_abs_sum(m);
    cl.sync();
    h_after = __fmul_rn(cluster_sum(cl, m.red + 1, nc), k.inv_B);
    if (A.trace && rank == 0 && tid == 0) { A.trace[2 * (n - 1)] = loss; A.trace[2 * (n - 1) + 1] = h_after; }
    const bool cont = (double)fabsf(h_after) > 0.88 * (double)fabsf(h_before) && n < A.max_steps;
    if (!cont) break;
    if (n >= A.rows - 1) { exhausted = true; break; }
  }
  // value_target <- value; write back the replica of rank 0 (all replicas are bit-identical)
  if (rank == 0) {
    for (int i = tid; i < NPARAM; i += NT) {
      const float p = m.P[smem_index(i)];
      A.params[i] = p;
      A.target[i] = p;
    }
#pragma unroll
    for (int q = 0; q < PER_T; ++q) {
      const int i = tid + q * NT;
      if (i < NPARAM) { A.exp_avg[i] = mom[q]; A.exp_avg_sq[i] = vel[q]; }
    }
    if (tid == 0) {
      *A.counter = cnt;
      A.out[0] = (float)n; A.out[1] = loss; A.out[2] = h_before; A.out[3] = h_after; A.out[4] = exhausted ? 1.f : 0.f;
    }
  }
  for (int i = tid; i < 2 * TS; i += NT) A.state[base * 2 + i] = m.x[i];
  cl.sync();   // no CTA leaves while another may still read its shared memory
}

constexpr size_t SMEM_BYTES = (size_t)SMEM_FLOATS * sizeof(float);

Consts make_consts(double gamma_atte, double th0, double th1, long long B) {
  Consts k;
  k.act_low[0] = -5.f; k.act_high[0] = 5.f;
  k.act_low[1] = (float)(-1.0 / gamma_atte); k.act_high[1] = (float)(1.0 / gamma_atte);
  k.th[0] = (float)th0; k.th[1] = (float)th1;
  k.dt = (float)(1.0 / 200.0);
  k.k3 = (float)(1.0 / (2.0 * gamma_atte * gamma_atte));
  k.gam2 = (float)(gamma_atte * gamma_atte);
  k.wcoef = (float)(0.5 / (gamma_atte * gamma_atte));
  k.inv_B = 1.f / (float)B;
  return k;
}

bool act_ok(int act) { return act >= GOPS_ACT_RELU && act <= GOPS_ACT_TANH; }

int smem_for(const void* fn, const void* p) { return gops::allow_smem(fn, gops::device_of(p), (int)SMEM_BYTES); }

}  // namespace

extern "C" {

int gops_b200_rpi_policy(const float* target_params, int32_t act, double gamma_atte, const float* obs, int64_t batch,
                         float* act_out, void* stream) {
  ENTRY();
  if (!target_params || !obs || !act_out) return fail("rpi_policy: null argument");
  if (batch <= 0) return fail("rpi_policy: batch must be positive");
  if (!act_ok(act)) return fail("rpi_policy: unsupported hidden activation");
  DevGuard dg(target_params);
  const Consts k = make_consts(gamma_atte, 0.0, 0.0, batch);
  const unsigned grid = (unsigned)((batch + TS - 1) / TS);
#define GOPS_RPI_POLICY(ACT)                                                                                      \
  do {                                                                                                           \
    if (smem_for((const void*)rpi_policy_kernel<ACT>, target_params)) return 1;                                  \
    rpi_policy_kernel<ACT><<<grid, NT, SMEM_BYTES, (cudaStream_t)stream>>>(target_params, obs, batch, k, act_out); \
  } while (0)
  GOPS_ACT_SWITCH(act, GOPS_RPI_POLICY);
#undef GOPS_RPI_POLICY
  ++g_launches;
  CUDA_OK(cudaGetLastError(), "rpi_policy launch");
  return 0;
}

int gops_b200_rpi_loss_grad(const float* params, int32_t act, double gamma_atte, const float* obs, const float* act_in,
                            int64_t batch, float* scratch, float* grad_out, float* loss_out, void* stream) {
  ENTRY();
  if (!params || !obs || !act_in || !scratch || !grad_out || !loss_out) return fail("rpi_loss_grad: null argument");
  if (batch <= 0 || batch % TS) return fail("rpi_loss_grad: batch must be a positive multiple of 64");
  if (!act_ok(act)) return fail("rpi_loss_grad: unsupported hidden activation");
  DevGuard dg(params);
  const Consts k = make_consts(gamma_atte, 0.0, 0.0, batch);
  const int tiles = (int)(batch / TS);
  float* part_g = scratch;
  float* part_l = scratch + (size_t)tiles * NPARAM;
#define GOPS_RPI_LOSS(ACT)                                                                                         \
  do {                                                                                                            \
    if (smem_for((const void*)rpi_loss_tile_kernel<ACT>, params)) return 1;                                       \
    rpi_loss_tile_kernel<ACT><<<tiles, NT, SMEM_BYTES, (cudaStream_t)stream>>>(params, obs, act_in, k, part_g, part_l); \
  } while (0)
  GOPS_ACT_SWITCH(act, GOPS_RPI_LOSS);
#undef GOPS_RPI_LOSS
  rpi_reduce_kernel<<<(NPARAM + 255) / 256, 256, 0, (cudaStream_t)stream>>>(part_g, part_l, tiles, k.inv_B, grad_out,
                                                                            loss_out);
  g_launches += 2;
  CUDA_OK(cudaGetLastError(), "rpi_loss_grad launch");
  return 0;
}

int64_t gops_b200_rpi_scratch_floats(int64_t batch) { return batch <= 0 ? 0 : ((batch + TS - 1) / TS) * (NPARAM + 1); }

int gops_b200_rpi_newton(float* params, float* target, float* exp_avg, float* exp_avg_sq, int64_t step0, double lr,
                         double beta1, double beta2, double eps, int32_t act, double gamma_atte, double threshold0, double threshold1,
                         float* state, const int32_t* max_step, int32_t* counter, const float* draws, int32_t rows,
                         int32_t max_steps, int64_t batch, float* out, float* trace, void* stream) {
  ENTRY();
  if (!params || !target || !exp_avg || !exp_avg_sq || !state || !max_step || !counter || !draws || !out)
    return fail("rpi_newton: null argument");
  if (batch <= 0 || batch % TS || batch > TS * MAX_CLUSTER)
    return fail("rpi_newton: batch must be a multiple of 64 and at most 512");
  if (!act_ok(act)) return fail("rpi_newton: unsupported hidden activation");
  if (max_steps < 1 || rows < 2) return fail("rpi_newton: need max_steps >= 1 and at least 2 rows of draws");
  if (step0 < 0) return fail("rpi_newton: negative Adam step");
  DevGuard dg(params);
  NewtonArgs a;
  a.params = params; a.target = target; a.exp_avg = exp_avg; a.exp_avg_sq = exp_avg_sq;
  a.state = state; a.max_step = max_step; a.counter = counter; a.draws = draws; a.rows = rows; a.max_steps = max_steps;
  a.step0 = step0; a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.out = out; a.trace = trace; a.B = batch;
  const Consts k = make_consts(gamma_atte, threshold0, threshold1, batch);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(batch / TS));
  cfg.blockDim = dim3(NT);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)(batch / TS);
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
#define GOPS_RPI_NEWTON(ACT)                                                                 \
  do {                                                                                      \
    if (smem_for((const void*)rpi_newton_kernel<ACT>, params)) return 1;                    \
    CUDA_OK(cudaLaunchKernelEx(&cfg, rpi_newton_kernel<ACT>, a, k), "rpi_newton launch");   \
  } while (0)
  GOPS_ACT_SWITCH(act, GOPS_RPI_NEWTON);
#undef GOPS_RPI_NEWTON
  ++g_launches;
  return 0;
}

}  // extern "C"
