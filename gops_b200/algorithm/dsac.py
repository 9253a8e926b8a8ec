"""Distributional Soft Actor-Critic (DSAC), H100 edition.

Same plugin surface as the reference (gops/algorithm/dsac.py: ApproxContainer :34-65, DSAC :68-290).  One update =
five network evaluations and three back-propagations, all on the layer-wise wgmma MLP (csrc/dense_tc.cu, BF16x3),
joined by the library's fused elementwise kernels (csrc/dsac.cu: reparameterised tanh-Gaussian sampling and its
log-density, clipped-TD distributional critic loss, actor loss -- each with its hand-derived gradient), the fused Adam
and Polyak kernels.  No autograd graph, no host round trip until the scalars of the update are read back.

Random numbers: the reference draws five standard-normal tensors per update from torch's global CPU generator
(`rsample` of the two action distributions, `normal.sample()` in the three `__q_evaluate` calls, of which only the
target-critic one is used).  Here the three that matter are drawn on the device (`torch.randn`, a per-algorithm
generator); `noise_override = {"eps_new", "eps_next", "z_next"}` injects given tensors instead -- the parity protocol
of tests/test_gpu_dsac.py, which replays the noise recorded from the unmodified reference."""
__all__ = ["DSAC"]

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
    """One stochastic policy, one distributional action value, their Polyak targets and the temperature."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        q_args = get_apprfunc_dict("value", **kwargs)
        self.q = create_apprfunc(**q_args)
        self.q_target = target_copy(self.q)
        policy_args = get_apprfunc_dict("policy", **kwargs)
        self.policy = create_apprfunc(**policy_args)
        self.policy_target = target_copy(self.policy)
        self.log_alpha = nn.Parameter(torch.tensor(1, dtype=torch.float32))
        self.q_optimizer = FusedAdam(self.q.flat_params, lr=kwargs["value_learning_rate"])
        self.policy_optimizer = FusedAdam(self.policy.flat_params, lr=kwargs["policy_learning_rate"])
        # the temperature is ONE scalar: torch.optim.Adam's arithmetic on it runs on the host in fp32 (ScalarAdam)
        self.alpha_optimizer = ScalarAdam(self.log_alpha, lr=kwargs["alpha_learning_rate"])
        self.optimizer_dict = {"q": self.q_optimizer, "policy": self.policy_optimizer}
        self.scheduler_dict = {}

    def create_action_distributions(self, logits):
        return self.policy.get_act_dist(logits)


class DSAC(SoftActorCritic):
    _critics = ("q",)
    _policy_target = True
    _noise_shapes = (("eps_new", "BA"), ("eps_next", "BA"), ("z_next", "B"))
    _n_out = 8

    def __init__(self, index=0, **kwargs):
        super().__init__(index, **kwargs)
        self.networks = ApproxContainer(**kwargs)
        self.gamma = kwargs["gamma"]
        self.tau = kwargs["tau"]
        self.target_entropy = -kwargs["action_dim"]
        self.auto_alpha = kwargs["auto_alpha"]
        self.alpha = kwargs.get("alpha", 0.2)
        self.bound = kwargs["bound"]
        self.delay_update = kwargs["delay_update"]
        self._init_soft_ac(kwargs)

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "auto_alpha", "alpha", "bound", "delay_update")

    def _critic_buffers(self, B: int, z) -> dict:
        return dict(q_out=z(B, 2), q2_out=z(B, 2), qn_out=z(B, 2), dq=z(B, 2), dqn=z(B, 2), stats=z(2 * B))

    def _losses(self, b, n_q, n_qT, rew, done, noise, alpha):
        L, P, st = _lib.lib(), _lib.ptr, _lib.stream_ptr
        B, A, O = b["B"], self.act_dim, self.obs_dim
        q, pol = self.networks.q, self.networks.policy
        # critic: loss on (obs, act) against the clipped TD target from q_target(obs2, act2)
        n_q.forward(b["qin"], slot=0, train=True, out=b["q_out"])
        n_qT.forward(b["qin2"], train=False, out=b["q2_out"])
        _lib.check(L.gops_b200_dsac_q_loss(P(b["q_out"]), P(b["q2_out"]), P(noise["z_next"]), P(b["logp2"]), P(rew),
                                           P(done), B, float(self.gamma), float(alpha), int(bool(self.bound)),
                                           P(b["dq"]), P(b["out"]), st()))
        n_q.backward(b["dq"], slot=0, grad=self._grad_view(q))
        # actor: alpha logp - q(obs, new_act), back through the (frozen) critic into the policy
        n_q.forward(b["qin_new"], slot=1, train=True, out=b["qn_out"])
        _lib.check(L.gops_b200_dsac_policy_loss(P(b["qn_out"]), P(b["logp_new"]), B, float(alpha),
                                                float(self.target_entropy), P(b["dqn"]), P(b["out"][3:]), P(b["stats"]),
                                                st()))
        d_qin = n_q.backward(b["dqn"], slot=1, grad=None, want_dx=True)
        _lib.check(L.gops_b200_dsac_sample_backward(P(b["logits"]), P(noise["eps_new"]), B, A, float(pol.min_log_std),
                                                    float(pol.max_log_std), P(b["half"]), P(d_qin), O + A, O,
                                                    float(alpha) / B, P(b["dlogits"]), st()))

    def _tb(self, h, alpha):
        # h = [loss_q, mean q, mean q_std, loss_policy, entropy, mean(logp + H_target), pol mean, pol std]
        if self.auto_alpha:         # loss_alpha = -log_alpha * mean(logp + target_entropy)   (dsac.py:272-278)
            self.networks.alpha_optimizer.grad = -h[5]
        return {
            "DSAC/critic_avg_q-RL iter": h[1], "DSAC/critic_avg_std-RL iter": h[2],
            tb_tags["loss_actor"]: h[3], "DSAC/policy_mean-RL iter": h[6], "DSAC/policy_std-RL iter": h[7],
            "DSAC/entropy-RL iter": h[4], "DSAC/alpha-RL iter": alpha,
            tb_tags["loss_critic"]: h[0],
        }
