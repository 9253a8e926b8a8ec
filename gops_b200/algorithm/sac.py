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

import time
from copy import deepcopy
from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from gops_b200 import _lib
from gops_b200.algorithm.base import AlgorithmBase, ApprBase
from gops_b200.create_pkg.create_apprfunc import create_apprfunc
from gops_b200.ops.layerwise_mlp import layerwise_pair
from gops_b200.utils.common_utils import get_apprfunc_dict
from gops_b200.utils.flat_params import FusedAdam, ScalarAdam, polyak_update
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
        self.q1_target = deepcopy(self.q1)
        self.q2_target = deepcopy(self.q2)
        for net in (self.q1_target, self.q2_target):
            net.__dict__["_flat_params"] = type(self.q1.flat_params)(getattr(net, net._attr))
            net.__dict__["_nets"] = {}
            for p in net.parameters():
                p.requires_grad = False
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


class SAC(AlgorithmBase):
    def __init__(self, index: int = 0, gamma: float = 0.99, tau: float = 0.005, auto_alpha: bool = True,
                 alpha: float = 0.2, target_entropy: Optional[float] = None, **kwargs: Any):
        super().__init__(index, **kwargs)
        self.networks = ApproxContainer(**kwargs)
        self.gamma = gamma
        self.tau = tau
        self.auto_alpha = auto_alpha
        self.alpha = alpha
        self.target_entropy = -kwargs["action_dim"] if target_entropy is None else target_entropy
        self.obs_dim, self.act_dim = kwargs["obsv_dim"], kwargs["action_dim"]
        self.noise_override: Optional[Dict[str, torch.Tensor]] = None
        self._gen = None
        self._buf = {}
        if torch.cuda.is_available():
            self.networks.cuda()

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "auto_alpha", "alpha", "target_entropy")

    # ------------------------------------------------------------------------------------------------ plugin surface
    def local_update(self, data: dict, iteration: int) -> dict:
        tb_info = self.__compute_gradient(data, iteration)
        self.__update(iteration)
        return tb_info

    def get_remote_update_info(self, data: dict, iteration: int) -> Tuple[dict, dict]:
        tb_info = self.__compute_gradient(data, iteration)
        nets = self.networks
        update_info = {"q1_grad": [p._grad for p in nets.q1.parameters()],
                       "q2_grad": [p._grad for p in nets.q2.parameters()],
                       "policy_grad": [p._grad for p in nets.policy.parameters()], "iteration": iteration}
        if self.auto_alpha:
            update_info["log_alpha_grad"] = nets.alpha_optimizer.grad
        return tb_info, update_info

    def remote_update(self, update_info: dict):
        nets = self.networks
        for key, mod in (("q1_grad", nets.q1), ("q2_grad", nets.q2), ("policy_grad", nets.policy)):
            for p, grad in zip(mod.parameters(), update_info[key]):
                p._grad = grad
        if self.auto_alpha:
            nets.alpha_optimizer.grad = update_info["log_alpha_grad"]
        self.__update(update_info["iteration"])

    # ------------------------------------------------------------------------------------------------ internals
    def _device(self) -> torch.device:
        p = next(self.networks.q1.parameters())
        if not p.is_cuda:
            if not torch.cuda.is_available():
                raise RuntimeError("gops_b200: no CUDA device -- the SAC update has no CPU fallback")
            self.networks.cuda()
            p = next(self.networks.q1.parameters())
        return p.device

    def __get_alpha(self) -> float:
        return float(np.exp(np.float32(self.networks.log_alpha.item()))) if self.auto_alpha else self.alpha

    def _buffers(self, B: int, dev) -> dict:
        b = self._buf
        if b.get("B") != B or b.get("dev") != dev:
            A, O = self.act_dim, self.obs_dim
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
            b = self._buf = dict(B=B, dev=dev, logits=z(B, 2 * A), logits2=z(B, 2 * A), act_new=z(B, A), act2=z(B, A),
                                 logp_new=z(B), logp2=z(B), qin=z(B, O + A), qin_new=z(B, O + A), qin2=z(B, O + A),
                                 q=z(2, B, 1), qn=z(2, B, 1), qt=z(2, B, 1), dq=z(2, B, 1), dqn=z(2, B, 1),
                                 dlogits=z(B, 2 * A), out=z(6), host=torch.zeros(6).pin_memory())
            pol = self.networks.policy
            b["half"] = ((pol.act_high_lim - pol.act_low_lim) / 2).to(dev, torch.float32).contiguous()
            b["mid"] = ((pol.act_high_lim + pol.act_low_lim) / 2).to(dev, torch.float32).contiguous()
        return b

    def _noise(self, B: int, dev):
        if self.noise_override is not None:
            n = self.noise_override
            return (n["eps_new"].to(dev, torch.float32).reshape(B, self.act_dim).contiguous(),
                    n["eps_next"].to(dev, torch.float32).reshape(B, self.act_dim).contiguous())
        if self._gen is None or self._gen.device != dev:
            self._gen = torch.Generator(device=dev).manual_seed(int(torch.initial_seed() % (2 ** 31)))
        r = lambda *s: torch.randn(*s, generator=self._gen, device=dev, dtype=torch.float32)
        return r(B, self.act_dim), r(B, self.act_dim)

    def __compute_gradient(self, data: dict, iteration: int) -> dict:
        start_time = time.time()
        dev = self._device()
        nets, L, P = self.networks, _lib.lib(), _lib.ptr
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        obs, act, rew, obs2, done = (f32(data[k]) for k in ("obs", "act", "rew", "obs2", "done"))
        B, A, O = obs.shape[0], self.act_dim, self.obs_dim
        act = act.reshape(B, A)
        b = self._buffers(B, dev)
        eps_new, eps_next = self._noise(B, dev)
        alpha = self.__get_alpha()
        pol = nets.policy
        n_pol = pol.layerwise(B, 2, "train")           # slot 0: obs (trained), slot 1: obs2 (target action)
        n_q = layerwise_pair(nets.q1, nets.q2, B, 2, "train")
        n_qT = layerwise_pair(nets.q1_target, nets.q2_target, B, 1, "infer")
        for net, mod in ((n_pol, pol), (n_q.a, nets.q1), (n_q.b, nets.q2), (n_qT.a, nets.q1_target),
                         (n_qT.b, nets.q2_target)):
            net.pack(mod.flat_params.sync())
        lo, hi = float(pol.min_log_std), float(pol.max_log_std)
        q, qn, qt, dq, dqn = b["q"], b["qn"], b["qt"], b["dq"], b["dqn"]
        st = _lib.stream_ptr
        with torch.cuda.device(dev):
            # new action for the actor loss, next action for the critic target (sac.py:161-164, 215-218)
            n_pol.forward(obs, slot=0, train=True, out=b["logits"])
            _lib.check(L.gops_b200_dsac_sample(P(b["logits"]), P(eps_new), B, A, lo, hi, P(b["half"]), P(b["mid"]),
                                               P(b["act_new"]), P(b["logp_new"]), P(obs), O, P(b["qin_new"]), O + A,
                                               None, st()))
            n_pol.forward(obs2, slot=1, train=False, out=b["logits2"])
            _lib.check(L.gops_b200_dsac_sample(P(b["logits2"]), P(eps_next), B, A, lo, hi, P(b["half"]), P(b["mid"]),
                                               P(b["act2"]), P(b["logp2"]), P(obs2), O, P(b["qin2"]), O + A, None, st()))
            # the three twin-critic evaluations, all with the pre-update weights, then every loss in one kernel
            b["qin"][:, :O].copy_(obs)
            b["qin"][:, O:].copy_(act)
            n_q.forward(b["qin"], slot=0, train=True, out_a=q[0], out_b=q[1])
            n_q.forward(b["qin_new"], slot=1, train=True, out_a=qn[0], out_b=qn[1])
            n_qT.forward(b["qin2"], train=False, out_a=qt[0], out_b=qt[1])
            _lib.check(L.gops_b200_sac_losses(P(q[0]), P(q[1]), P(qn[0]), P(qn[1]), P(qt[0]), P(qt[1]), P(b["logp_new"]),
                                              P(b["logp2"]), P(rew), P(done), B, float(self.gamma), float(alpha),
                                              float(self.target_entropy), P(dq[0]), P(dq[1]), P(dqn[0]), P(dqn[1]),
                                              P(b["out"]), st()))
            # critics: weight gradients of the soft-Q loss at (obs, act)
            grads = []
            for net in (nets.q1, nets.q2):
                net.flat_params.bind_grads()
                grads.append(net.flat_params.gbuf[:net.flat_params.gbuf.numel() - 4])
            n_q.backward(dq[0], dq[1], slot=0, grad_a=grads[0], grad_b=grads[1])
            # actor: back through the (frozen) critics at (obs, new_act) and the sample into the policy
            dx1, dx2 = n_q.backward(dqn[0], dqn[1], slot=1, want_dx=True)
            _lib.check(L.gops_b200_dsact_sample_backward(P(b["logits"]), P(eps_new), B, A, lo, hi, P(b["half"]), P(dx1),
                                                         P(dx2), O + A, O, float(alpha) / B, P(b["dlogits"]), st()))
            pol.flat_params.bind_grads()
            n_pol.backward(b["dlogits"], slot=0, grad=pol.flat_params.gbuf[:pol.flat_params.gbuf.numel() - 4])
            b["host"].copy_(b["out"], non_blocking=True)
            torch.cuda.current_stream().synchronize()
        # [loss_q, mean q1, mean q2, loss_policy, entropy, d loss_alpha / d log_alpha]
        h = b["host"].tolist()
        if self.auto_alpha:         # loss_alpha = -log_alpha * mean(logp + target_entropy)   (sac.py:236-241)
            nets.alpha_optimizer.grad = h[5]
        return {
            tb_tags["loss_critic"]: h[0], tb_tags["loss_actor"]: h[3],
            "SAC/critic_avg_q1-RL iter": h[1], "SAC/critic_avg_q2-RL iter": h[2],
            "SAC/entropy-RL iter": h[4], "SAC/alpha-RL iter": alpha,
            tb_tags["alg_time"]: (time.time() - start_time) * 1000,
        }

    def __update(self, iteration: int):
        nets = self.networks
        nets.q1_optimizer.step()
        nets.q2_optimizer.step()
        nets.policy_optimizer.step()
        if self.auto_alpha:
            nets.alpha_optimizer.step()
        polyak_update(nets.q1_target.flat_params, nets.q1.flat_params, self.tau)
        polyak_update(nets.q2_target.flat_params, nets.q2.flat_params, self.tau)
