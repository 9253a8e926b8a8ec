"""DSAC-T (DSACT), the refined DSAC with twin distributional critics, H100 edition.

Same plugin surface as the reference (gops/algorithm/dsact.py: ApproxContainer :34-74, DSACT :77-358).  One update =
two policy evaluations and three evaluations of the twin critics (online at (obs, act) and (obs, new_act), targets at
(obs2, act2)), each twin evaluation a PAIRED pass of the layer-wise wgmma MLP (csrc/dense_tc.cu, mlpnet_pair_*): both
critics in every layer launch, so the twins cost the launches of one network.  Between them: the tanh-Gaussian sampling
kernels shared with DSAC (csrc/dsac.cu) and the DSAC-T loss kernels (csrc/dsact.cu: twin critic loss with the running
mean of the critics' std, twin-min actor loss, sample gradient summed over both critics), then the fused Adam and
Polyak kernels.  No autograd graph; one host read-back of the update's scalars.

Random numbers: the reference draws eight standard-normal tensors per update from torch's global CPU generator, of
which four reach a result (the two action samples and the two target-critic samples).  Here those four are drawn on the
device (`torch.randn`, a per-algorithm generator); `noise_override = {"eps_new", "eps_next", "z1_next", "z2_next"}`
injects given tensors instead.

`mean_std1` / `mean_std2`, the running means of the critics' std (not part of the state_dict, as in the reference),
live on the device; reading them returns the value after the last update (None before the first), assigning them
(e.g. to resume from a reference run) takes effect at the next update."""
__all__ = ["ApproxContainer", "DSACT"]

from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from gops_b200 import _lib
from gops_b200.algorithm._soft_ac import SoftActorCritic
from gops_b200.algorithm.base import ApprBase, target_copy
from gops_b200.create_pkg.create_apprfunc import create_apprfunc
from gops_b200.utils.common_utils import get_apprfunc_dict
from gops_b200.utils.flat_params import FusedAdam, ScalarAdam
from gops_b200.utils.tensorboard_setup import tb_tags


class ApproxContainer(ApprBase):
    """One stochastic policy, two distributional action values, their Polyak targets and the temperature."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        q_args = get_apprfunc_dict("value", **kwargs)
        self.q1 = create_apprfunc(**q_args)
        self.q2 = create_apprfunc(**q_args)
        self.q1_target = target_copy(self.q1)
        self.q2_target = target_copy(self.q2)
        policy_args = get_apprfunc_dict("policy", **kwargs)
        self.policy = create_apprfunc(**policy_args)
        self.policy_target = target_copy(self.policy)
        self.log_alpha = nn.Parameter(torch.tensor(1, dtype=torch.float32))
        self.q1_optimizer = FusedAdam(self.q1.flat_params, lr=kwargs["value_learning_rate"])
        self.q2_optimizer = FusedAdam(self.q2.flat_params, lr=kwargs["value_learning_rate"])
        self.policy_optimizer = FusedAdam(self.policy.flat_params, lr=kwargs["policy_learning_rate"])
        # the temperature is ONE scalar: torch.optim.Adam's arithmetic on it runs on the host in fp32 (ScalarAdam)
        self.alpha_optimizer = ScalarAdam(self.log_alpha, lr=kwargs["alpha_learning_rate"])
        self.optimizer_dict = {"q1": self.q1_optimizer, "q2": self.q2_optimizer, "policy": self.policy_optimizer}
        self.scheduler_dict = {}

    def create_action_distributions(self, logits):
        return self.policy.get_act_dist(logits)


class DSACT(SoftActorCritic):
    _critics = ("q1", "q2")
    _policy_target = True
    _noise_shapes = (("eps_new", "BA"), ("eps_next", "BA"), ("z1_next", "B"), ("z2_next", "B"))
    _n_out = 14

    def __init__(self, index=0, **kwargs):
        super().__init__(index, **kwargs)
        self.networks = ApproxContainer(**kwargs)
        self.gamma = kwargs["gamma"]
        self.tau = kwargs["tau"]
        self.target_entropy = -kwargs["action_dim"]
        self.auto_alpha = kwargs["auto_alpha"]
        self.alpha = kwargs.get("alpha", 0.2)
        self.delay_update = kwargs["delay_update"]
        self.tau_b = kwargs.get("tau_b", self.tau)
        self._mean_std_dev = None                   # device float[2], the running means the kernels update
        self._mean_std = [None, None]               # their host values after the last update (None = unset)
        self._init_soft_ac(kwargs)

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "auto_alpha", "alpha", "delay_update")

    # running means of the critics' std (dsact.py:243-251)
    @property
    def mean_std1(self) -> Optional[float]:
        return self._mean_std[0]

    @mean_std1.setter
    def mean_std1(self, value):
        self._set_mean_std(0, value)

    @property
    def mean_std2(self) -> Optional[float]:
        return self._mean_std[1]

    @mean_std2.setter
    def mean_std2(self, value):
        self._set_mean_std(1, value)

    def _set_mean_std(self, i: int, value):
        self._mean_std[i] = None if value is None else float(np.float32(float(value)))
        if value is not None and self._mean_std_dev is not None:
            self._mean_std_dev[i] = self._mean_std[i]

    def _mean_std_buffer(self, dev) -> torch.Tensor:
        if self._mean_std_dev is None or self._mean_std_dev.device != dev:
            self._mean_std_dev = torch.tensor([0.0 if m is None else m for m in self._mean_std], dtype=torch.float32,
                                              device=dev)
        return self._mean_std_dev

    def _critic_buffers(self, B: int, z) -> dict:
        return dict(q1_out=z(B, 2), q2_out=z(B, 2), t1_out=z(B, 2), t2_out=z(B, 2), qn1_out=z(B, 2), qn2_out=z(B, 2),
                    dq1=z(B, 2), dq2=z(B, 2), dqn1=z(B, 2), dqn2=z(B, 2), stats=z(2 * B))

    def _losses(self, b, n_q, n_qT, rew, done, noise, alpha):
        L, P, st = _lib.lib(), _lib.ptr, _lib.stream_ptr
        B, A, O = b["B"], self.act_dim, self.obs_dim
        nets, pol = self.networks, self.networks.policy
        mean_std = self._mean_std_buffer(b["dev"])
        unset = int(self._mean_std[0] is None) | (int(self._mean_std[1] is None) << 1)
        # critics: twin loss on (obs, act) against the targets' TD samples at (obs2, act2)
        n_q.forward(b["qin"], slot=0, train=True, out_a=b["q1_out"], out_b=b["q2_out"])
        n_qT.forward(b["qin2"], train=False, out_a=b["t1_out"], out_b=b["t2_out"])
        _lib.check(L.gops_b200_dsact_q_loss(P(b["q1_out"]), P(b["q2_out"]), P(b["t1_out"]), P(b["t2_out"]),
                                            P(noise["z1_next"]), P(noise["z2_next"]), P(b["logp2"]), P(rew), P(done), B,
                                            float(self.gamma), float(alpha), float(self.tau_b), P(mean_std), unset,
                                            P(b["dq1"]), P(b["dq2"]), P(b["out"]), st()))
        n_q.backward(b["dq1"], b["dq2"], slot=0, grad_a=self._grad_view(nets.q1), grad_b=self._grad_view(nets.q2))
        # actor: alpha logp - min(q1, q2)(obs, new_act), back through the (frozen) critics into the policy
        n_q.forward(b["qin_new"], slot=1, train=True, out_a=b["qn1_out"], out_b=b["qn2_out"])
        _lib.check(L.gops_b200_dsact_policy_loss(P(b["qn1_out"]), P(b["qn2_out"]), P(b["logp_new"]), B, float(alpha),
                                                 float(self.target_entropy), P(b["dqn1"]), P(b["dqn2"]),
                                                 P(b["out"][9:]), P(b["stats"]), st()))
        dx1, dx2 = n_q.backward(b["dqn1"], b["dqn2"], slot=1, want_dx=True)
        _lib.check(L.gops_b200_dsact_sample_backward(P(b["logits"]), P(noise["eps_new"]), B, A, float(pol.min_log_std),
                                                     float(pol.max_log_std), P(b["half"]), P(dx1), P(dx2), O + A, O,
                                                     float(alpha) / B, P(b["dlogits"]), st()))

    def _tb(self, h, alpha):
        # h = [loss_q, q1, q2, std1, std2, min std1, min std2, mean_std1, mean_std2,
        #      loss_policy, entropy, mean(logp + H_target), pol mean, pol std]
        self._mean_std = [h[7], h[8]]
        if self.auto_alpha:         # loss_alpha = -log_alpha * mean(logp + target_entropy)   (dsact.py:323-329)
            self.networks.alpha_optimizer.grad = -h[11]
        return {
            "DSAC2/critic_avg_q1-RL iter": h[1], "DSAC2/critic_avg_q2-RL iter": h[2],
            "DSAC2/critic_avg_std1-RL iter": h[3], "DSAC2/critic_avg_std2-RL iter": h[4],
            "DSAC2/critic_avg_min_std1-RL iter": h[5], "DSAC2/critic_avg_min_std2-RL iter": h[6],
            tb_tags["loss_actor"]: h[9], tb_tags["loss_critic"]: h[0],
            "DSAC2/policy_mean-RL iter": h[12], "DSAC2/policy_std-RL iter": h[13],
            "DSAC2/entropy-RL iter": h[10], "DSAC2/alpha-RL iter": alpha,
            "DSAC2/mean_std1": h[7], "DSAC2/mean_std2": h[8],
        }
