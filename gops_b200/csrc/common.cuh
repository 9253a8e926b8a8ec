// Device-side helpers shared by the gops_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gops_b200.h"

namespace gops {

constexpr int MAXA = GOPS_B200_MAX_ACT;
constexpr int LQN = GOPS_B200_MAX_LQ_N;
constexpr int kMaxObs = 16;     // observation entries with ClipObservation bounds (state==obs models: pyth_mobilerobot has 13)

// ---------------------------------------------------------------------------------------------
// mbarrier + TMA (cp.async.bulk) primitives: weights are staged global -> shared by the bulk-copy
// engine (SASS: UBLKCP) and signalled through an mbarrier transaction count.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// Activations (gops/utils/common_utils.py:26-55 -> torch.nn.{ReLU,ELU,GELU,SELU,Sigmoid,Tanh,Identity})
// h = g(x), d = g'(x) in fp32 with the accurate libdevice functions (no fast-math).
// ---------------------------------------------------------------------------------------------
// Exact-erf GELU with ONE exponential shared by the Gaussian cdf and pdf:
//   e = exp(-x^2/2);  erfc(|x|/sqrt2) = e * P(k), k = 1/(1 + p |x|/sqrt2)   (Abramowitz-Stegun 7.1.26, |err| <= 1.5e-7)
//   cdf = x >= 0 ? 1 - 0.5 e P : 0.5 e P;   pdf = e / sqrt(2 pi);   gelu = x cdf;   gelu' = cdf + x pdf
// ~20 instructions instead of libdevice erff + expf (~45); the parity tests bound the effect on loss / gradient.
__device__ __forceinline__ void gelu_parts(float x, float& cdf, float& pdf) {
  const float ax = fabsf(x);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * x * -0.72134752044448170368f));   // exp(-x^2/2)
  float k;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(k) : "f"(fmaf(ax, 0.23164189045f, 1.0f)));      // p / sqrt(2) = 0.2316419
  float pl = fmaf(1.061405429f, k, -1.453152027f);
  pl = fmaf(pl, k, 1.421413741f);
  pl = fmaf(pl, k, -0.284496736f);
  pl = fmaf(pl, k, 0.254829592f);
  const float half_erfc = 0.5f * (pl * k) * e;
  cdf = x >= 0.f ? 1.f - half_erfc : half_erfc;
  pdf = 0.39894228040143267794f * e;
}

// ---------------------------------------------------------------------------------------------
// FP32 pairs: the epilogues process adjacent columns as (lo, hi) pairs held in one 64-bit register pair.  sm_90 has no
// packed FP32 arithmetic, so each pair operation is two scalar IEEE-rn operations in the same order (the pair form keeps
// the epilogue code shared and lets the compiler interleave the two independent chains).
// ---------------------------------------------------------------------------------------------
namespace f32x2 {
typedef unsigned long long u64;
__device__ __forceinline__ u64 pk(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void upk(u64 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ u64 fma(u64 a, u64 b, u64 c) {
  float a0, a1, b0, b1, c0, c1;
  upk(a, a0, a1); upk(b, b0, b1); upk(c, c0, c1);
  return pk(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ u64 mul(u64 a, u64 b) {
  float a0, a1, b0, b1;
  upk(a, a0, a1); upk(b, b0, b1);
  return pk(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ u64 add(u64 a, u64 b) {
  float a0, a1, b0, b1;
  upk(a, a0, a1); upk(b, b0, b1);
  return pk(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64 rep(float c) { return pk(c, c); }
__device__ __forceinline__ u64 ld(const float* p) { return *reinterpret_cast<const u64*>(p); }      // 8-byte aligned pair
}  // namespace f32x2

// gelu_parts for a pair: H = x cdf, D = cdf + x pdf (WANT_D).  0.5 is folded into the polynomial (an exact scaling).
template <bool WANT_D>
__device__ __forceinline__ void gelu_pair(f32x2::u64 X, f32x2::u64& H, f32x2::u64& D) {
  using namespace f32x2;
  float x0, x1, a0, a1, e0, e1, k0, k1;
  upk(X, x0, x1);
  upk(mul(mul(X, X), rep(-0.72134752044448170368f)), a0, a1);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(a0));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(a1));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(k0) : "f"(fmaf(fabsf(x0), 0.23164189045f, 1.0f)));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(k1) : "f"(fmaf(fabsf(x1), 0.23164189045f, 1.0f)));
  const u64 K = pk(k0, k1), E = pk(e0, e1);
  u64 PL = fma(rep(0.5f * 1.061405429f), K, rep(0.5f * -1.453152027f));
  PL = fma(PL, K, rep(0.5f * 1.421413741f));
  PL = fma(PL, K, rep(0.5f * -0.284496736f));
  PL = fma(PL, K, rep(0.5f * 0.254829592f));
  const u64 HE = mul(mul(PL, K), E);                 // half erfc(|x| / sqrt 2)
  float he0, he1, q0, q1;
  upk(HE, he0, he1);
  upk(fma(HE, rep(-1.f), rep(1.f)), q0, q1);
  const u64 CDF = pk(x0 >= 0.f ? q0 : he0, x1 >= 0.f ? q1 : he1);
  H = mul(X, CDF);
  if constexpr (WANT_D) D = fma(X, mul(E, rep(0.39894228040143267794f)), CDF);
}

__device__ __forceinline__ float act_fwd(int act, float x) {
  switch (act) {
    case GOPS_ACT_RELU: return fmaxf(x, 0.f);
    case GOPS_ACT_ELU: return x > 0.f ? x : expm1f(x);
    case GOPS_ACT_GELU: { float c, q; gelu_parts(x, c, q); return x * c; }
    case GOPS_ACT_SELU: return 1.0507009873554805f * (x > 0.f ? x : 1.6732632423543772f * expm1f(x));
    case GOPS_ACT_SIGMOID: return 1.f / (1.f + expf(-x));
    case GOPS_ACT_TANH: return tanhf(x);
    default: return x;
  }
}
__device__ __forceinline__ void act_fwd_grad(int act, float x, float& h, float& d) {
  switch (act) {
    case GOPS_ACT_RELU: h = fmaxf(x, 0.f); d = x > 0.f ? 1.f : 0.f; break;
    case GOPS_ACT_ELU:
      if (x > 0.f) { h = x; d = 1.f; } else { float e = expf(x); h = expm1f(x); d = e; }
      break;
    case GOPS_ACT_GELU: {
      float cdf, pdf;
      gelu_parts(x, cdf, pdf);
      h = x * cdf; d = cdf + x * pdf;
    } break;
    case GOPS_ACT_SELU: {
      const float sc = 1.0507009873554805f, al = 1.6732632423543772f;
      if (x > 0.f) { h = sc * x; d = sc; } else { h = sc * al * expm1f(x); d = sc * al * expf(x); }
    } break;
    case GOPS_ACT_SIGMOID: h = 1.f / (1.f + expf(-x)); d = h * (1.f - h); break;
    case GOPS_ACT_TANH: h = tanhf(x); d = 1.f - h * h; break;
    default: h = x; d = 1.f; break;
  }
}

// Compile-time activation variants: the per-element `switch (act)` of act_fwd / act_fwd_grad is a branch region per
// element, which stops the compiler from interleaving independent elements (every element then costs its full
// dependent-chain latency).  Hot loops dispatch ONCE on the activation id and run a loop specialised on ACT.
template <int ACT>
__device__ __forceinline__ float act_fwd_t(float x) {
  if constexpr (ACT == GOPS_ACT_RELU) return fmaxf(x, 0.f);
  else if constexpr (ACT == GOPS_ACT_ELU) return x > 0.f ? x : expm1f(x);
  else if constexpr (ACT == GOPS_ACT_GELU) { float c, q; gelu_parts(x, c, q); return x * c; }
  else if constexpr (ACT == GOPS_ACT_SELU) return 1.0507009873554805f * (x > 0.f ? x : 1.6732632423543772f * expm1f(x));
  else if constexpr (ACT == GOPS_ACT_SIGMOID) return 1.f / (1.f + expf(-x));
  else if constexpr (ACT == GOPS_ACT_TANH) return tanhf(x);
  else return x;
}
template <int ACT>
__device__ __forceinline__ void act_fwd_grad_t(float x, float& h, float& d) {
  if constexpr (ACT == GOPS_ACT_RELU) { h = fmaxf(x, 0.f); d = x > 0.f ? 1.f : 0.f; }
  else if constexpr (ACT == GOPS_ACT_ELU) {
    const float e = expf(x), em = expm1f(x);
    h = x > 0.f ? x : em; d = x > 0.f ? 1.f : e;
  } else if constexpr (ACT == GOPS_ACT_GELU) {
    float cdf, pdf;
    gelu_parts(x, cdf, pdf);
    h = x * cdf; d = cdf + x * pdf;
  } else if constexpr (ACT == GOPS_ACT_SELU) {
    const float sc = 1.0507009873554805f, al = 1.6732632423543772f;
    const float e = expf(x), em = expm1f(x);
    h = x > 0.f ? sc * x : sc * al * em; d = x > 0.f ? sc : sc * al * e;
  } else if constexpr (ACT == GOPS_ACT_SIGMOID) { h = 1.f / (1.f + expf(-x)); d = h * (1.f - h); }
  else if constexpr (ACT == GOPS_ACT_TANH) { h = tanhf(x); d = 1.f - h * h; }
  else { h = x; d = 1.f; }
}
// Pair forms (adjacent columns): GELU runs packed, the others are two scalar evaluations.
template <int ACT>
__device__ __forceinline__ void act_fwd_pair_t(f32x2::u64 X, float& h0, float& h1) {
  if constexpr (ACT == GOPS_ACT_GELU) {
    f32x2::u64 Hh, D;
    gelu_pair<false>(X, Hh, D);
    f32x2::upk(Hh, h0, h1);
  } else {
    float x0, x1;
    f32x2::upk(X, x0, x1);
    h0 = act_fwd_t<ACT>(x0);
    h1 = act_fwd_t<ACT>(x1);
  }
}
template <int ACT>
__device__ __forceinline__ void act_fwd_grad_pair_t(f32x2::u64 X, float& h0, float& h1, float& d0, float& d1) {
  if constexpr (ACT == GOPS_ACT_GELU) {
    f32x2::u64 Hh, D;
    gelu_pair<true>(X, Hh, D);
    f32x2::upk(Hh, h0, h1);
    f32x2::upk(D, d0, d1);
  } else {
    float x0, x1;
    f32x2::upk(X, x0, x1);
    act_fwd_grad_t<ACT>(x0, h0, d0);
    act_fwd_grad_t<ACT>(x1, h1, d1);
  }
}
// GOPS_ACT_SWITCH(act, M): expands M(ACT) for the runtime activation id `act` (M is a one-argument macro)
#define GOPS_ACT_SWITCH(act, M)                 \
  switch (act) {                                \
    case GOPS_ACT_RELU: M(GOPS_ACT_RELU); break;       \
    case GOPS_ACT_ELU: M(GOPS_ACT_ELU); break;         \
    case GOPS_ACT_GELU: M(GOPS_ACT_GELU); break;       \
    case GOPS_ACT_SELU: M(GOPS_ACT_SELU); break;       \
    case GOPS_ACT_SIGMOID: M(GOPS_ACT_SIGMOID); break; \
    case GOPS_ACT_TANH: M(GOPS_ACT_TANH); break;       \
    default: M(GOPS_ACT_LINEAR); break;                \
  }

// angle_normalize, gops/utils/math_utils.py:8-11: ((x + pi) % (2 pi)) - pi with floored modulo,
// evaluated in fp32 like torch.remainder on a float32 tensor.
__device__ __forceinline__ float angle_normalize(float x) {
  const float PI_F = 3.14159265358979323846f, TWO_PI_F = 6.28318530717958647692f;
  float y = __fadd_rn(x, PI_F);
  float r = fmodf(y, TWO_PI_F);
  if (r != 0.f && r < 0.f) r = __fadd_rn(r, TWO_PI_F);
  return __fsub_rn(r, PI_F);
}

}  // namespace gops
