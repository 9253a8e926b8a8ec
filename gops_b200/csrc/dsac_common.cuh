// Device helpers shared by the DSAC (dsac.cu), DSAC-T (dsact.cu) and SAC (sac.cu) elementwise kernels: the
// ActionValueDistri head, fixed-order block reductions, the soft TD target, the twin-min gradient and the gradient of
// the reparameterised tanh-Gaussian sample.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace gops {
namespace dsac {

constexpr float kEps = 1e-6f;                    // act_distribution_type.py:15 EPS
constexpr float kHalfLog2Pi = 0.91893853320467274178f;

// q head of ActionValueDistri (mlp.py:289-296): mean | softplus(raw)
__device__ __forceinline__ float softplus(float x) { return x > 20.f ? x : log1pf(expf(x)); }   // torch threshold 20
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

// reduction over the batch in fixed order: each of the 256 threads folds a strided range sequentially, then a fixed
// tree.  Called by all threads of a 256-thread block; every thread gets the result.
template <class F, class Op>
__device__ float block_reduce(long long B, float init, F f, Op op) {
  __shared__ float sm[256];
  float s = init;
  for (long long i = threadIdx.x; i < B; i += 256) s = op(s, f(i));
  sm[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sm[threadIdx.x] = op(sm[threadIdx.x], sm[threadIdx.x + o]);
    __syncthreads();
  }
  const float r = sm[0];
  __syncthreads();
  return r;
}
template <class F>
__device__ float block_sum(long long B, F f) {
  return block_reduce(B, 0.f, f, [](float a, float b) { return a + b; });
}

// r + (1 - d) gamma (q - alpha logp), in the reference's operation order
__device__ __forceinline__ float td_target(float r, float d, float gamma, float q, float alpha, float logp) {
  return __fadd_rn(r, __fmul_rn(__fmul_rn(__fsub_rn(1.f, d), gamma), __fsub_rn(q, __fmul_rn(alpha, logp))));
}

// Gradient g of min(a, b) split as torch.minimum's backward does: all of it to the smaller value, half to each on a
// tie, zero to the larger.
__device__ __forceinline__ void twin_min_grad(float a, float b, float g, float& ga, float& gb) {
  ga = a < b ? g : a == b ? 0.5f * g : 0.f;
  gb = b < a ? g : a == b ? 0.5f * g : 0.f;
}

// d loss / d logits of one sample of the policy net, given dA(j) = d loss / d act_j and the coefficient c of log p in
// the loss:   loss = ... + c * sum_b logp_b
template <class DA>
__device__ __forceinline__ void sample_bwd_row(const float* __restrict__ logits, const float* __restrict__ eps, long long b,
                                               int A, float lo, float hi, const float* __restrict__ half, float c, DA dA,
                                               float* __restrict__ dlogits) {
  for (int j = 0; j < A; ++j) {
    const float mean = logits[b * 2 * A + j], raw = logits[b * 2 * A + A + j];
    const float ls = fminf(fmaxf(raw, lo), hi), sd = expf(ls), e = eps[b * A + j];
    const float u = mean + sd * e, t = tanhf(u), om = 1.f - t * t;
    // act = half t + mid;   -log(1 + EPS - t^2) has derivative 2 t (1 - t^2) / (1 + EPS - t^2) w.r.t. u
    const float du = dA(j) * half[j] * om + c * (2.f * t * om / (1.f + kEps - t * t));
    const float dls = (du * e * sd - c) * ((raw >= lo && raw <= hi) ? 1.f : 0.f);   // d(-log std)/d ls = -1
    dlogits[b * 2 * A + j] = du;
    dlogits[b * 2 * A + A + j] = dls;
  }
}

}  // namespace dsac
}  // namespace gops
