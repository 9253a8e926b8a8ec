// Small non-template kernels (packing, partial reduction, Adam, Polyak); included by gops_b200.cu only.
#pragma once
#include "rollout.cuh"

#include "adam_math.cuh"

namespace gops {

// ---------------------------------------------------------------------------------------------
// torch-layout flat parameters -> packed k-major blob (W1^T, W2^T with row stride HP; 16-byte aligned parts)
// ---------------------------------------------------------------------------------------------
__global__ void pack_params_kernel(const float* __restrict__ flat, NetL L, int HID, float* __restrict__ blob) {
  const int HP = HID == 64 ? 72 : HID + 4;
  const bool split = HID == 64;          // 64-wide nets: hi / lo planes for the 3xTF32 tensor-core GEMMs
  const int n = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  const float* W1 = flat + L.g_w1;
  const float* W2 = flat + L.g_w2;
  const float* W3 = flat + L.g_w3;
  const int rows1 = split ? L.in8 : L.in;
  for (int i = t0; i < rows1 * HP; i += n) {       // W1^T, k-major, row stride HP (pad rows / columns = 0)
    const int k = i / HP, o = i - k * HP;
    const float w = (o < HID && k < L.in) ? W1[o * L.in + k] : 0.f;
    if (split) {
      uint32_t hi;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(w));
      const int is = k * HP + (o < HID ? (o ^ (((k >> 2) & 1) << 2)) : o);   // bank swizzle, see gemm_fwd_mma
      blob[L.o_w1 + is] = __uint_as_float(hi);
      blob[L.o_w1l + is] = w - __uint_as_float(hi);
    } else {
      blob[L.o_w1 + i] = w;
    }
  }
  for (int i = t0; i < HID * HP; i += n) {         // W2^T
    const int k = i / HP, o = i - k * HP;
    const float w = o < HID ? W2[o * HID + k] : 0.f;
    if (split) {
      uint32_t hi;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(w));
      const int is = k * HP + (o < HID ? (o ^ (((k >> 2) & 1) << 2)) : o);
      blob[L.o_w2 + is] = __uint_as_float(hi);
      blob[L.o_w2l + is] = w - __uint_as_float(hi);
    } else {
      blob[L.o_w2 + i] = w;
    }
  }
  for (int i = t0; i < L.out * HID; i += n) blob[L.o_w3 + i] = W3[i];
  for (int i = t0; i < HID; i += n) {
    blob[L.o_b1 + i] = flat[L.g_b1 + i];
    blob[L.o_b2 + i] = flat[L.g_b2 + i];
  }
  for (int i = t0; i < 4; i += n) blob[L.o_b3 + i] = i < L.out ? flat[L.g_b3 + i] : 0.f;
}

// grad[i] = sum_c partial[c][i] in fixed CTA order; the 3 trailing scalars go to scalars_out
__global__ void reduce_partials_kernel(const float* __restrict__ partial, int n_cta, int stride, int nparam,
                                       float* __restrict__ grad, float* __restrict__ scalars) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nparam + 4) return;
  float s = 0.f;
  for (int c = 0; c < n_cta; ++c) s += partial[(size_t)c * stride + i];
  if (i < nparam) {
    if (grad) grad[i] = s;
  } else if (scalars) {
    scalars[i - nparam] = s;
  }
}

// torch.optim.Adam, single tensor path (torch/optim/adam.py _single_tensor_adam, no amsgrad/decay)
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, long long n, float omb1, float b2, float omb2, float eps,
                            float step_size, float bc2_sqrt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float pi = p[i], mi = m[i], vi = v[i];
  adam_update(g[i], pi, mi, vi, omb1, b2, omb2, eps, step_size, bc2_sqrt);
  p[i] = pi;
  m[i] = mi;
  v[i] = vi;
}

// SPIL's PI multiplier controller (spil.py:257-270), one thread per constraint, between the value and policy passes.
// tail: the value pass's reduced scalars (slots 2 / 3 = safe trajectories of constraint 0 / 1, summed over ranks).
// st: float64 [delta_i(2), safe_prob_pre(2), lam(2)], updated in place.  w: float32 [w_r, w_c0, w_c1] for the policy pass.
// The float64 arithmetic is written with explicit _rn intrinsics (no FMA contraction) so that it equals the NumPy
// expression bit for bit; safe_prob is a float32 mean and (safe_prob_pre - safe_prob) a float32 difference, as the
// reference's float32 arrays make them, and Kd * delta_d is a float32 product (python scalar times a float32 array).
__global__ void spil_controller_kernel(const float* __restrict__ tail, long long batch, double kp, double ki, float kd,
                                       double thr0, double thr1, double* __restrict__ st, float* __restrict__ w) {
  __shared__ double lam_s[2];
  // np.clip: a NaN stays NaN
  auto clip = [](double x, double hi) { return x < 0.0 ? 0.0 : (x > hi ? hi : x); };
  const int i = threadIdx.x;
  if (i < 2) {
    const float sp = __fdiv_rn(tail[2 + i], (float)batch);
    const double dp = __dadd_rn(i == 0 ? thr0 : thr1, -(double)sp);
    const double adp = fabs(dp);
    double sep = adp > 0.1 ? __dmul_rn(dp, 0.7) : dp;       // integral separation
    if (adp > 0.2) sep = __dmul_rn(dp, 0.0);
    const double di = clip(__dadd_rn(st[i], sep), 99999.0);
    const float dd = (float)clip((double)__fsub_rn((float)st[2 + i], sp), 3333.0);
    const double l = clip(__dadd_rn(__dadd_rn(__dmul_rn(ki, di), __dmul_rn(kp, dp)), (double)__fmul_rn(kd, dd)), 3333.0);
    st[i] = di;
    st[2 + i] = (double)sp;
    st[4 + i] = l;
    lam_s[i] = l;
  }
  __syncthreads();
  if (i < 2) {
    const double den = __dadd_rn(1.0, __dadd_rn(lam_s[0], lam_s[1]));
    if (i == 0) w[0] = (float)__ddiv_rn(1.0, den);
    w[1 + i] = (float)__ddiv_rn(lam_s[i], den);
  }
}

__global__ void polyak_kernel(float* __restrict__ tgt, const float* __restrict__ src, float tau, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) tgt[i] = tgt[i] * (1.f - tau) + tau * src[i];
}

}  // namespace gops
