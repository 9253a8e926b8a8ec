// Elementwise half of the SAC update (reference gops/algorithm/sac.py:159-241): the twin soft-Q loss, the twin-min
// actor loss and the temperature gradient in ONE kernel, each with its hand-derived gradient towards the critic outputs.
// The reference takes no optimizer step between its critic and actor losses, so both read critics with the same
// (pre-update) weights and one kernel can follow all three paired critic forwards of an update (dense_tc.cu,
// mlpnet_pair_*).  Action sampling is gops_b200_dsac_sample, the action gradient gops_b200_dsact_sample_backward.
// All reductions are fixed-order (deterministic).
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

// q1 / q2: the critics at (obs, act); qn1 / qn2: at (obs, new_act); t1 / t2: the target critics at (obs2, next_act).
//   y = r + (1 - d) gamma (min(t1, t2) - alpha logp_next)                 (sac.py:204-226)
//   loss_q = mean((q1 - y)^2) + mean((q2 - y)^2)                           dq_i = 2 (q_i - y) / B
//   loss_pi = mean(alpha logp_new - min(qn1, qn2))                        (sac.py:228-234)
//   d loss_alpha / d log_alpha = -mean(logp_new + target_entropy)         (sac.py:236-241)
// One block of 256 threads.  out: [0] loss_q, [1] mean q1, [2] mean q2, [3] loss_pi, [4] entropy = -mean(logp_new),
// [5] the log_alpha gradient.
__global__ void sac_losses_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                  const float* __restrict__ qn1, const float* __restrict__ qn2,
                                  const float* __restrict__ t1, const float* __restrict__ t2,
                                  const float* __restrict__ logp_new, const float* __restrict__ logp_next,
                                  const float* __restrict__ rew, const float* __restrict__ done, long long B, float gamma,
                                  float alpha, float target_entropy, float* __restrict__ dq1, float* __restrict__ dq2,
                                  float* __restrict__ dqn1, float* __restrict__ dqn2, float* __restrict__ out) {
  const float invB = 1.f / (float)B;
  const auto td = [&](long long i) { return td_target(rew[i], done[i], gamma, fminf(t1[i], t2[i]), alpha, logp_next[i]); };
  const float l1 = block_sum(B, [&](long long i) {
    const float e = q1[i] - td(i);
    dq1[i] = 2.f * e * invB;
    return e * e;
  }) / (float)B;
  const float l2 = block_sum(B, [&](long long i) {
    const float e = q2[i] - td(i);
    dq2[i] = 2.f * e * invB;
    return e * e;
  }) / (float)B;
  const float mq1 = block_sum(B, [&](long long i) { return q1[i]; }) / (float)B;
  const float mq2 = block_sum(B, [&](long long i) { return q2[i]; }) / (float)B;
  const float lp = block_sum(B, [&](long long i) {
    const float a = qn1[i], b = qn2[i];
    twin_min_grad(a, b, -invB, dqn1[i], dqn2[i]);
    return alpha * logp_new[i] - fminf(a, b);
  }) / (float)B;
  const float ml = block_sum(B, [&](long long i) { return logp_new[i]; }) / (float)B;
  const float mh = block_sum(B, [&](long long i) { return logp_new[i] + target_entropy; }) / (float)B;
  if (threadIdx.x == 0) { out[0] = l1 + l2; out[1] = mq1; out[2] = mq2; out[3] = lp; out[4] = -ml; out[5] = -mh; }
}

}  // namespace

extern "C" {

int gops_b200_sac_losses(const float* q1_out, const float* q2_out, const float* q1_new_out, const float* q2_new_out,
                         const float* q1_next_out, const float* q2_next_out, const float* logp_new,
                         const float* logp_next, const float* rew, const float* done, int64_t batch, float gamma,
                         float alpha, float target_entropy, float* d_q1_out, float* d_q2_out, float* d_q1_new_out,
                         float* d_q2_new_out, float* out6, void* stream) {
  if (!q1_out || !q2_out || !q1_new_out || !q2_new_out || !q1_next_out || !q2_next_out || !logp_new || !logp_next ||
      !rew || !done || !d_q1_out || !d_q2_out || !d_q1_new_out || !d_q2_new_out || !out6 || batch < 1)
    return fail("sac_losses: bad argument");
  DevGuard dg(q1_out);
  sac_losses_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(q1_out, q2_out, q1_new_out, q2_new_out, q1_next_out,
                                                        q2_next_out, logp_new, logp_next, rew, done, batch, gamma, alpha,
                                                        target_entropy, d_q1_out, d_q2_out, d_q1_new_out, d_q2_new_out,
                                                        out6);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError(), "sac kernel");
  return 0;
}

}  // extern "C"
