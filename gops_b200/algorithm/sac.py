"""SAC (Soft Actor-Critic), H100 edition.

Same plugin surface as the reference (gops/algorithm/sac.py: ApproxContainer :32-71, SAC :74-263).  One update = two
policy evaluations (obs for the actor's action, obs2 for the target action: SAC has no policy target) and three
evaluations of the twin ActionValue critics (online at (obs, act) and (obs, new_act), targets at (obs2, next_act)),
each twin evaluation a PAIRED pass of the layer-wise wgmma MLP (csrc/dense_tc.cu, mlpnet_pair_*).  The reference takes
no optimizer step between its critic and actor losses, so all three read the pre-update weights and ONE kernel
(csrc/sac.cu) then forms both losses, the temperature gradient and every output gradient.  Action sampling and the
action gradient through both critics are DSAC's / DSAC-T's kernels; then the fused Adam and Polyak kernels.  No
autograd graph; one host read-back of the update's scalars.

Random numbers: the reference draws two standard-normal tensors per update from torch's global CPU generator (eps_new
for the actor's action, then eps_next for the target action).  Here they are drawn on the device (`torch.randn`, a
per-algorithm generator); `noise_override = {"eps_new", "eps_next"}` injects given tensors instead.  Unlike the
reference, the update does not write new_act / new_logp into `data`."""
__all__ = ["ApproxContainer", "SAC"]

from typing import Any, Optional

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
    """One stochastic policy, two action values, their Polyak targets and the temperature."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        q_args = get_apprfunc_dict("value", **kwargs)
        self.q1 = create_apprfunc(**q_args)
        self.q2 = create_apprfunc(**q_args)
        policy_args = get_apprfunc_dict("policy", **kwargs)
        self.policy = create_apprfunc(**policy_args)
        self.q1_target = target_copy(self.q1)
        self.q2_target = target_copy(self.q2)
        self.log_alpha = nn.Parameter(torch.tensor(1, dtype=torch.float32))
        self.q1_optimizer = FusedAdam(self.q1.flat_params, lr=kwargs["q_learning_rate"])
        self.q2_optimizer = FusedAdam(self.q2.flat_params, lr=kwargs["q_learning_rate"])
        self.policy_optimizer = FusedAdam(self.policy.flat_params, lr=kwargs["policy_learning_rate"])
        # the temperature is ONE scalar: torch.optim.Adam's arithmetic on it runs on the host in fp32 (ScalarAdam)
        self.alpha_optimizer = ScalarAdam(self.log_alpha, lr=kwargs["alpha_learning_rate"])
        self.optimizer_dict = {"q1": self.q1_optimizer, "q2": self.q2_optimizer, "policy": self.policy_optimizer}
        self.scheduler_dict = {}

    def create_action_distributions(self, logits):
        return self.policy.get_act_dist(logits)


class SAC(SoftActorCritic):
    _critics = ("q1", "q2")
    _policy_target = False
    _noise_shapes = (("eps_new", "BA"), ("eps_next", "BA"))
    _n_out = 6
    delay_update = 1              # the policy, the temperature and the critics' targets move on every update

    def __init__(self, index: int = 0, gamma: float = 0.99, tau: float = 0.005, auto_alpha: bool = True,
                 alpha: float = 0.2, target_entropy: Optional[float] = None, **kwargs: Any):
        super().__init__(index, **kwargs)
        self.networks = ApproxContainer(**kwargs)
        self.gamma = gamma
        self.tau = tau
        self.auto_alpha = auto_alpha
        self.alpha = alpha
        self.target_entropy = -kwargs["action_dim"] if target_entropy is None else target_entropy
        self._init_soft_ac(kwargs)

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "auto_alpha", "alpha", "target_entropy")

    def _critic_buffers(self, B: int, z) -> dict:
        return dict(q=z(2, B, 1), qn=z(2, B, 1), qt=z(2, B, 1), dq=z(2, B, 1), dqn=z(2, B, 1))

    def _losses(self, b, n_q, n_qT, rew, done, noise, alpha):
        L, P, st = _lib.lib(), _lib.ptr, _lib.stream_ptr
        B, A, O = b["B"], self.act_dim, self.obs_dim
        nets, pol = self.networks, self.networks.policy
        q, qn, qt, dq, dqn = b["q"], b["qn"], b["qt"], b["dq"], b["dqn"]
        # the three twin-critic evaluations, all with the pre-update weights, then every loss in one kernel
        n_q.forward(b["qin"], slot=0, train=True, out_a=q[0], out_b=q[1])
        n_q.forward(b["qin_new"], slot=1, train=True, out_a=qn[0], out_b=qn[1])
        n_qT.forward(b["qin2"], train=False, out_a=qt[0], out_b=qt[1])
        _lib.check(L.gops_b200_sac_losses(P(q[0]), P(q[1]), P(qn[0]), P(qn[1]), P(qt[0]), P(qt[1]), P(b["logp_new"]),
                                          P(b["logp2"]), P(rew), P(done), B, float(self.gamma), float(alpha),
                                          float(self.target_entropy), P(dq[0]), P(dq[1]), P(dqn[0]), P(dqn[1]),
                                          P(b["out"]), st()))
        # critics: weight gradients of the soft-Q loss at (obs, act)
        n_q.backward(dq[0], dq[1], slot=0, grad_a=self._grad_view(nets.q1), grad_b=self._grad_view(nets.q2))
        # actor: back through the (frozen) critics at (obs, new_act) and the sample into the policy
        dx1, dx2 = n_q.backward(dqn[0], dqn[1], slot=1, want_dx=True)
        _lib.check(L.gops_b200_dsact_sample_backward(P(b["logits"]), P(noise["eps_new"]), B, A, float(pol.min_log_std),
                                                     float(pol.max_log_std), P(b["half"]), P(dx1), P(dx2), O + A, O,
                                                     float(alpha) / B, P(b["dlogits"]), st()))

    def _tb(self, h, alpha):
        # h = [loss_q, mean q1, mean q2, loss_policy, entropy, d loss_alpha / d log_alpha]
        if self.auto_alpha:         # loss_alpha = -log_alpha * mean(logp + target_entropy)   (sac.py:236-241)
            self.networks.alpha_optimizer.grad = h[5]
        return {
            tb_tags["loss_critic"]: h[0], tb_tags["loss_actor"]: h[3],
            "SAC/critic_avg_q1-RL iter": h[1], "SAC/critic_avg_q2-RL iter": h[2],
            "SAC/entropy-RL iter": h[4], "SAC/alpha-RL iter": alpha,
        }
