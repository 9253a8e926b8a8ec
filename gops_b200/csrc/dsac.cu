// Elementwise half of the DSAC update (reference gops/algorithm/dsac.py:155-290): everything between the network
// evaluations -- reparameterised tanh-Gaussian action sampling with its log-density (act_distribution_type.py:18-50),
// the distributional critic loss with the clipped TD target (dsac.py:219-262), the actor loss (dsac.py:264-270) -- each
// with its hand-derived gradient towards the network outputs.  The network evaluations themselves run on the
// layer-wise wgmma MLP (dense_tc.cu).  All reductions are fixed-order (deterministic).
#include "gops_b200.h"

#include <cuda_runtime.h>
#include <math.h>

#include <string>

#include "dsac_common.cuh"
#include "host_util.h"

using gops::DevGuard;
using gops::fail;

namespace {

using namespace gops::dsac;

// StochaPolicy head (mlp.py:203-221, std_type "mlp_shared") + TanhGaussDistribution.rsample (:37-50):
//   mean | log_std = logits;  std = exp(clamp(log_std, lo, hi));  u = mean + std eps;  a = half tanh(u) + mid
//   log p = sum_j [-eps^2/2 - log std - log sqrt(2 pi)] - sum_j log(1 + EPS - tanh(u)^2) - sum_j log(half)
// Writes act [B][A], logp [B] and, if qin != nullptr, the critic input row [obs | act] (ldq floats per row).
__global__ void dsac_sample_kernel(const float* __restrict__ logits, const float* __restrict__ eps, long long B, int A,
                                   float lo, float hi, const float* __restrict__ half, const float* __restrict__ mid,
                                   float* __restrict__ act, float* __restrict__ logp, const float* __restrict__ obs,
                                   int obs_dim, float* __restrict__ qin, int ldq, float* __restrict__ stats) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float lp = 0.f;
  for (int j = 0; j < A; ++j) {
    const float mean = logits[b * 2 * A + j], ls = fminf(fmaxf(logits[b * 2 * A + A + j], lo), hi);
    const float sd = expf(ls), e = eps[b * A + j];
    const float u = mean + sd * e, t = tanhf(u);
    const float a = half[j] * t + mid[j];
    act[b * A + j] = a;
    if (qin) qin[b * ldq + obs_dim + j] = a;
    lp += (-(e * e) * 0.5f - ls - kHalfLog2Pi) - logf(1.f + kEps - t * t) - logf(half[j]);
  }
  logp[b] = lp;
  if (qin)
    for (int f = 0; f < obs_dim; ++f) qin[b * ldq + f] = obs[b * obs_dim + f];
  if (stats) {   // tb: tanh(mean_0), std_0 of every sample (reduced by the caller's scalar pass)
    stats[b] = tanhf(logits[b * 2 * A]);
    stats[B + b] = expf(fminf(fmaxf(logits[b * 2 * A + A], lo), hi));
  }
}

// d loss / d logits of the policy net, given dA = d loss / d act [B][ldda] (columns a0 .. a0 + A - 1) and the
// coefficient c of log p in the loss (alpha / B):   loss = ... + c * sum_b logp_b
__global__ void dsac_sample_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ eps, long long B, int A,
                                       float lo, float hi, const float* __restrict__ half, const float* __restrict__ dA,
                                       int ldda, int a0, float c, float* __restrict__ dlogits) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  sample_bwd_row(logits, eps, b, A, lo, hi, half, c, [&](int j) { return dA[b * ldda + a0 + j]; }, dlogits);
}

// Critic loss (dsac.py:219-262, bound = True):
//   q, q_std = head(qo);  q_next = mean2 + clamp(z2, -3, 3) * std2 (q_target on (obs2, act2))
//   target = r + (1 - d) gamma (q_next - alpha logp2);  bound = 3 mean(q_std)
//   target_b = q + clamp(target - q, -bound, bound)
//   loss = mean[(q - target)^2 / (2 q_std_det^2) + (q_det - target_b)^2 / (2 q_std^2) + log q_std]
// One block (the batch is a minibatch: 8192): pass 1 mean(q_std), pass 2 loss + gradient w.r.t. the critic outputs.
// out: [0] loss, [1] mean q, [2] mean q_std.
__global__ void dsac_q_loss_kernel(const float* __restrict__ qo, const float* __restrict__ qo2, const float* __restrict__ z2,
                                   const float* __restrict__ logp2, const float* __restrict__ rew,
                                   const float* __restrict__ done, long long B, float gamma, float alpha, int bound,
                                   float* __restrict__ dqo, float* __restrict__ out) {
  const float invB = 1.f / (float)B;
  const float mstd = block_sum(B, [&](long long i) { return softplus(qo[2 * i + 1]); }) * invB;
  const float mq = block_sum(B, [&](long long i) { return qo[2 * i]; }) * invB;
  const float tdb = 3.f * mstd;
  const float loss = block_sum(B, [&](long long i) {
    const float q = qo[2 * i], raw = qo[2 * i + 1], sd = softplus(raw);
    const float zz = fminf(fmaxf(z2[i], -3.f), 3.f);
    const float qn = qo2[2 * i] + zz * softplus(qo2[2 * i + 1]);
    const float target = rew[i] + (1.f - done[i]) * gamma * (qn - alpha * logp2[i]);
    float l, dq, dsd;
    if (bound) {
      const float tb = q + fminf(fmaxf(target - q, -tdb), tdb);
      const float e1 = q - target, e2 = q - tb;
      l = e1 * e1 / (2.f * sd * sd) + e2 * e2 / (2.f * sd * sd) + logf(sd);
      dq = e1 / (sd * sd);                      // the second term holds q.detach() and the detached target_b
      dsd = -e2 * e2 / (sd * sd * sd) + 1.f / sd;   // the first term holds q_std.detach()
    } else {                                    // -Normal(q, q_std).log_prob(target)
      const float e1 = q - target;
      l = e1 * e1 / (2.f * sd * sd) + logf(sd) + kHalfLog2Pi;
      dq = e1 / (sd * sd);
      dsd = -e1 * e1 / (sd * sd * sd) + 1.f / sd;
    }
    dqo[2 * i] = dq * invB;
    dqo[2 * i + 1] = dsd * sigmoidf(raw) * invB;
    return l;
  }) * invB;
  if (threadIdx.x == 0) { out[0] = loss; out[1] = mq; out[2] = mstd; }
}

// Actor loss (dsac.py:264-270): mean(alpha logp_new - q(obs, new_act)); gradient towards the critic output is -1/B on
// the mean column.  out: [0] loss, [1] entropy = -mean(logp_new), [2] mean(logp_new + target_entropy) (alpha loss).
__global__ void dsac_policy_loss_kernel(const float* __restrict__ qo, const float* __restrict__ logp, long long B,
                                        float alpha, float target_entropy, float* __restrict__ dqo,
                                        float* __restrict__ out, const float* __restrict__ stats) {
  const float invB = 1.f / (float)B;
  const float l = block_sum(B, [&](long long i) {
    dqo[2 * i] = -invB;
    dqo[2 * i + 1] = 0.f;
    return alpha * logp[i] - qo[2 * i];
  }) * invB;
  const float ml = block_sum(B, [&](long long i) { return logp[i]; }) * invB;
  float pm = 0.f, ps = 0.f;
  if (stats) {
    pm = block_sum(B, [&](long long i) { return stats[i]; }) * invB;
    ps = block_sum(B, [&](long long i) { return stats[B + i]; }) * invB;
  }
  if (threadIdx.x == 0) { out[0] = l; out[1] = -ml; out[2] = ml + target_entropy; out[3] = pm; out[4] = ps; }
}

}  // namespace

extern "C" {

int gops_b200_dsac_sample(const float* logits, const float* eps, int64_t batch, int32_t act_dim, float min_log_std,
                          float max_log_std, const float* act_half, const float* act_mid, float* act, float* logp,
                          const float* obs, int32_t obs_dim, float* qin, int32_t ldq, float* stats, void* stream) {
  if (!logits || !eps || !act || !logp || !act_half || !act_mid || batch < 1 || act_dim < 1)
    return fail("dsac_sample: bad argument");
  DevGuard dg(logits);
  dsac_sample_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      logits, eps, batch, act_dim, min_log_std, max_log_std, act_half, act_mid, act, logp, obs, obs_dim, qin, ldq, stats);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError(), "dsac kernel");
  return 0;
}

int gops_b200_dsac_sample_backward(const float* logits, const float* eps, int64_t batch, int32_t act_dim, float min_log_std,
                                   float max_log_std, const float* act_half, const float* d_act, int32_t ldda,
                                   int32_t act_col0, float logp_coeff, float* d_logits, void* stream) {
  if (!logits || !eps || !d_act || !d_logits || !act_half || batch < 1) return fail("dsac_sample_backward: bad argument");
  DevGuard dg(logits);
  dsac_sample_bwd_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      logits, eps, batch, act_dim, min_log_std, max_log_std, act_half, d_act, ldda, act_col0, logp_coeff, d_logits);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError(), "dsac kernel");
  return 0;
}

int gops_b200_dsac_q_loss(const float* q_out, const float* q_next_out, const float* z_next, const float* logp_next,
                          const float* rew, const float* done, int64_t batch, float gamma, float alpha, int32_t bound,
                          float* d_q_out, float* out3, void* stream) {
  if (!q_out || !q_next_out || !z_next || !logp_next || !rew || !done || !d_q_out || !out3 || batch < 1)
    return fail("dsac_q_loss: bad argument");
  DevGuard dg(q_out);
  dsac_q_loss_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q_out, q_next_out, z_next, logp_next, rew, done, batch, gamma, alpha,
                                                         bound, d_q_out, out3);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError(), "dsac kernel");
  return 0;
}

int gops_b200_dsac_policy_loss(const float* q_out, const float* logp_new, int64_t batch, float alpha, float target_entropy,
                               float* d_q_out, float* out5, const float* stats, void* stream) {
  if (!q_out || !logp_new || !d_q_out || !out5 || batch < 1) return fail("dsac_policy_loss: bad argument");
  DevGuard dg(q_out);
  dsac_policy_loss_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q_out, logp_new, batch, alpha, target_entropy, d_q_out, out5,
                                                              stats);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError(), "dsac kernel");
  return 0;
}

}  // extern "C"
