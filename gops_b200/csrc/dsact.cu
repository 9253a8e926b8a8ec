// Elementwise half of the DSAC-T update (reference gops/algorithm/dsact.py:162-329): the twin-critic loss with the
// running mean of the critics' std and the variance-scaled surrogate (dsact.py:229-313), the twin-min actor loss
// (:315-321) and the sample gradient summed over both critics -- each with its hand-derived gradient towards the network
// outputs.  The critic evaluations run as pairs on the layer-wise wgmma MLP (dense_tc.cu, mlpnet_pair_*); the action
// sampling is gops_b200_dsac_sample.  All reductions are fixed-order (deterministic).
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

constexpr float kBias = 0.1f;                    // dsact.py:286

// Twin critic loss (dsact.py:229-313).  q1o / q2o: critic outputs [B][2] (mean | raw std) at (obs, act); t1o / t2o:
// target-critic outputs at (obs2, act2); z1 / z2: standard-normal noise of the two target samples.
//   std_i = softplus(raw_i);  m_i = mean(std_i);  mean_std_i = (1 - tau_b) mean_std_i + tau_b m_i, or m_i if unset
//   s_i = mean_i' + clamp(z_i, -3, 3) std_i'      (target critics)
//   q_next = min(q1', q2');  q_next_sample = q1' < q2' ? s_1 : s_2
//   t = r + (1 - d) gamma (q_next - alpha logp2);  ts = the same with q_next_sample
//   tb_i = q_i + clamp(ts - q_i, -3 mean_std_i, 3 mean_std_i)
//   loss_i = (mean_std_i^2 + 0.1) mean(-(t - q_i) / (sd_i^2 + 0.1) q_i - ((q_i - tb_i)^2 - sd_i^2) / (sd_i^3 + 0.1) std_i)
// with sd_i = max(std_i, 0) and everything but the q_i / std_i factors detached.  One block of 256 threads.
// mean_std [2] is read and written in place; bit i of `unset` seeds mean_std[i] instead.
// out: [0] loss_1 + loss_2, [1] mean q1, [2] mean q2, [3] mean std1, [4] mean std2, [5] min std1, [6] min std2,
//      [7] mean_std1, [8] mean_std2 (after this update).
__global__ void dsact_q_loss_kernel(const float* __restrict__ q1o, const float* __restrict__ q2o,
                                    const float* __restrict__ t1o, const float* __restrict__ t2o,
                                    const float* __restrict__ z1, const float* __restrict__ z2,
                                    const float* __restrict__ logp2, const float* __restrict__ rew,
                                    const float* __restrict__ done, long long B, float gamma, float alpha, float keep,
                                    float tau_b, int unset, float* __restrict__ mean_std, float* __restrict__ dq1,
                                    float* __restrict__ dq2, float* __restrict__ out) {
  const float invB = 1.f / (float)B;
  const auto mn = [](float a, float b) { return fminf(a, b); };
  const float ms1 = block_sum(B, [&](long long i) { return softplus(q1o[2 * i + 1]); }) / (float)B;
  const float ms2 = block_sum(B, [&](long long i) { return softplus(q2o[2 * i + 1]); }) / (float)B;
  const float mq1 = block_sum(B, [&](long long i) { return q1o[2 * i]; }) / (float)B;
  const float mq2 = block_sum(B, [&](long long i) { return q2o[2 * i]; }) / (float)B;
  const float min1 = block_reduce(B, INFINITY, [&](long long i) { return softplus(q1o[2 * i + 1]); }, mn);
  const float min2 = block_reduce(B, INFINITY, [&](long long i) { return softplus(q2o[2 * i + 1]); }, mn);
  // the running means (dsact.py:243-251), detached
  const float m1 = (unset & 1) ? ms1 : __fadd_rn(__fmul_rn(keep, mean_std[0]), __fmul_rn(tau_b, ms1));
  const float m2 = (unset & 2) ? ms2 : __fadd_rn(__fmul_rn(keep, mean_std[1]), __fmul_rn(tau_b, ms2));
  const float bound1 = 3.f * m1, bound2 = 3.f * m2;
  const float c1 = (m1 * m1 + kBias) * invB, c2 = (m2 * m2 + kBias) * invB;
  // per-critic loss term (before the (mean_std^2 + 0.1) / B factor) and its gradient towards (mean, raw std)
  const auto term = [&](const float* qo, float* dqo, long long i, float t, float ts, float bound, float c) {
    const float q = qo[2 * i], raw = qo[2 * i + 1], sd = softplus(raw), sdc = fmaxf(sd, 0.f);
    const float tb = q + fminf(fmaxf(ts - q, -bound), bound);
    const float gq = -(t - q) / (sdc * sdc + kBias);
    const float e = q - tb;
    const float gs = -(e * e - sdc * sdc) / (sdc * sdc * sdc + kBias);
    dqo[2 * i] = c * gq;
    dqo[2 * i + 1] = c * gs * sigmoidf(raw);
    return gq * q + gs * sd;
  };
  // the two TD targets of sample i (dsact.py:254-282): from the min of the target means and from the sample of the
  // target critic with the smaller mean (torch.where(q1 < q2, ..): a tie picks q2)
  const auto targets = [&](long long i, float& t, float& ts) {
    const float n1 = t1o[2 * i], n2 = t2o[2 * i];
    const float smp1 = __fadd_rn(n1, __fmul_rn(fminf(fmaxf(z1[i], -3.f), 3.f), softplus(t1o[2 * i + 1])));
    const float smp2 = __fadd_rn(n2, __fmul_rn(fminf(fmaxf(z2[i], -3.f), 3.f), softplus(t2o[2 * i + 1])));
    t = td_target(rew[i], done[i], gamma, fminf(n1, n2), alpha, logp2[i]);
    ts = td_target(rew[i], done[i], gamma, n1 < n2 ? smp1 : smp2, alpha, logp2[i]);
  };
  const float s1 = block_sum(B, [&](long long i) {
    float t, ts;
    targets(i, t, ts);
    return term(q1o, dq1, i, t, ts, bound1, c1);
  });
  const float s2 = block_sum(B, [&](long long i) {
    float t, ts;
    targets(i, t, ts);
    return term(q2o, dq2, i, t, ts, bound2, c2);
  });
  if (threadIdx.x == 0) {
    const float l1 = (m1 * m1 + kBias) * (s1 / (float)B), l2 = (m2 * m2 + kBias) * (s2 / (float)B);
    out[0] = l1 + l2; out[1] = mq1; out[2] = mq2; out[3] = ms1; out[4] = ms2; out[5] = min1; out[6] = min2;
    out[7] = m1; out[8] = m2;
    mean_std[0] = m1;
    mean_std[1] = m2;
  }
}

// Twin-min actor loss (dsact.py:315-321): mean(alpha logp_new - min(q1, q2)) on the critic means at (obs, new_act).
// The gradient -1/B goes to the critic with the smaller mean, -1/(2B) to each on a tie (torch.minimum's backward); the
// other critic gets a zero row.  out: [0] loss, [1] entropy = -mean(logp_new), [2] mean(logp_new + target_entropy),
// [3] mean tanh(mean_0), [4] mean std_0 (from the sample kernel's stats).
__global__ void dsact_policy_loss_kernel(const float* __restrict__ q1o, const float* __restrict__ q2o,
                                         const float* __restrict__ logp, long long B, float alpha, float target_entropy,
                                         float* __restrict__ dq1, float* __restrict__ dq2, float* __restrict__ out,
                                         const float* __restrict__ stats) {
  const float invB = 1.f / (float)B;
  const float l = block_sum(B, [&](long long i) {
    const float a = q1o[2 * i], b = q2o[2 * i];
    float g1, g2;
    twin_min_grad(a, b, -invB, g1, g2);
    dq1[2 * i] = g1; dq1[2 * i + 1] = 0.f;
    dq2[2 * i] = g2; dq2[2 * i + 1] = 0.f;
    return alpha * logp[i] - fminf(a, b);
  }) * invB;
  const float ml = block_sum(B, [&](long long i) { return logp[i]; }) * invB;
  float pm = 0.f, ps = 0.f;
  if (stats) {
    pm = block_sum(B, [&](long long i) { return stats[i]; }) * invB;
    ps = block_sum(B, [&](long long i) { return stats[B + i]; }) * invB;
  }
  if (threadIdx.x == 0) { out[0] = l; out[1] = -ml; out[2] = ml + target_entropy; out[3] = pm; out[4] = ps; }
}

// d loss / d logits when the action feeds both critics: dA = dA_1 + dA_2 (columns a0 .. a0 + A - 1 of each)
__global__ void dsact_sample_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ eps, long long B, int A,
                                        float lo, float hi, const float* __restrict__ half, const float* __restrict__ dA1,
                                        const float* __restrict__ dA2, int ldda, int a0, float c,
                                        float* __restrict__ dlogits) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  sample_bwd_row(logits, eps, b, A, lo, hi, half, c,
                 [&](int j) { return dA1[b * ldda + a0 + j] + dA2[b * ldda + a0 + j]; }, dlogits);
}

}  // namespace

extern "C" {

int gops_b200_dsact_q_loss(const float* q1_out, const float* q2_out, const float* q1_next_out, const float* q2_next_out,
                           const float* z1_next, const float* z2_next, const float* logp_next, const float* rew,
                           const float* done, int64_t batch, float gamma, float alpha, double tau_b, float* mean_std,
                           int32_t mean_std_unset, float* d_q1_out, float* d_q2_out, float* out9, void* stream) {
  if (!q1_out || !q2_out || !q1_next_out || !q2_next_out || !z1_next || !z2_next || !logp_next || !rew || !done ||
      !mean_std || !d_q1_out || !d_q2_out || !out9 || batch < 1)
    return fail("dsact_q_loss: bad argument");
  DevGuard dg(q1_out);
  dsact_q_loss_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q1_out, q2_out, q1_next_out, q2_next_out, z1_next, z2_next,
                                                          logp_next, rew, done, batch, gamma, alpha, (float)(1.0 - tau_b),
                                                          (float)tau_b, mean_std_unset, mean_std, d_q1_out, d_q2_out, out9);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError(), "dsact kernel");
  return 0;
}

int gops_b200_dsact_policy_loss(const float* q1_out, const float* q2_out, const float* logp_new, int64_t batch, float alpha,
                                float target_entropy, float* d_q1_out, float* d_q2_out, float* out5, const float* stats,
                                void* stream) {
  if (!q1_out || !q2_out || !logp_new || !d_q1_out || !d_q2_out || !out5 || batch < 1)
    return fail("dsact_policy_loss: bad argument");
  DevGuard dg(q1_out);
  dsact_policy_loss_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q1_out, q2_out, logp_new, batch, alpha, target_entropy,
                                                               d_q1_out, d_q2_out, out5, stats);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError(), "dsact kernel");
  return 0;
}

int gops_b200_dsact_sample_backward(const float* logits, const float* eps, int64_t batch, int32_t act_dim,
                                    float min_log_std, float max_log_std, const float* act_half, const float* d_act_1,
                                    const float* d_act_2, int32_t ldda, int32_t act_col0, float logp_coeff,
                                    float* d_logits, void* stream) {
  if (!logits || !eps || !d_act_1 || !d_act_2 || !d_logits || !act_half || batch < 1 || act_dim < 1)
    return fail("dsact_sample_backward: bad argument");
  DevGuard dg(logits);
  dsact_sample_bwd_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      logits, eps, batch, act_dim, min_log_std, max_log_std, act_half, d_act_1, d_act_2, ldda, act_col0, logp_coeff,
      d_logits);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError(), "dsact kernel");
  return 0;
}

}  // extern "C"
