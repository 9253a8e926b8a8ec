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

import time
from copy import deepcopy
from typing import Dict, Optional, Tuple

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
    """One stochastic policy, two distributional action values, their Polyak targets and the temperature."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        q_args = get_apprfunc_dict("value", **kwargs)
        self.q1 = create_apprfunc(**q_args)
        self.q2 = create_apprfunc(**q_args)
        self.q1_target = deepcopy(self.q1)
        self.q2_target = deepcopy(self.q2)
        policy_args = get_apprfunc_dict("policy", **kwargs)
        self.policy = create_apprfunc(**policy_args)
        self.policy_target = deepcopy(self.policy)
        for net in (self.q1_target, self.q2_target, self.policy_target):
            net.__dict__["_flat_params"] = type(self.q1.flat_params)(getattr(net, net._attr))
            net.__dict__["_nets"] = {}
            for p in net.parameters():
                p.requires_grad = False
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


class DSACT(AlgorithmBase):
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
        self.obs_dim, self.act_dim = kwargs["obsv_dim"], kwargs["action_dim"]
        self.noise_override: Optional[Dict[str, torch.Tensor]] = None
        self._gen = None
        self._buf = {}
        self._mean_std_dev = None                   # device float[2], the running means the kernels update
        self._mean_std = [None, None]               # their host values after the last update (None = unset)
        if torch.cuda.is_available():
            self.networks.cuda()

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
                raise RuntimeError("gops_b200: no CUDA device -- the DSAC-T update has no CPU fallback")
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
                                 q1_out=z(B, 2), q2_out=z(B, 2), t1_out=z(B, 2), t2_out=z(B, 2), qn1_out=z(B, 2),
                                 qn2_out=z(B, 2), dq1=z(B, 2), dq2=z(B, 2), dqn1=z(B, 2), dqn2=z(B, 2),
                                 dlogits=z(B, 2 * A), stats=z(2 * B), out=z(14), host=torch.zeros(14).pin_memory())
            pol = self.networks.policy
            b["half"] = ((pol.act_high_lim - pol.act_low_lim) / 2).to(dev, torch.float32).contiguous()
            b["mid"] = ((pol.act_high_lim + pol.act_low_lim) / 2).to(dev, torch.float32).contiguous()
        return b

    def _noise(self, B: int, dev):
        if self.noise_override is not None:
            n = self.noise_override
            return (n["eps_new"].to(dev, torch.float32).reshape(B, self.act_dim).contiguous(),
                    n["eps_next"].to(dev, torch.float32).reshape(B, self.act_dim).contiguous(),
                    n["z1_next"].to(dev, torch.float32).reshape(B).contiguous(),
                    n["z2_next"].to(dev, torch.float32).reshape(B).contiguous())
        if self._gen is None or self._gen.device != dev:
            self._gen = torch.Generator(device=dev).manual_seed(int(torch.initial_seed() % (2 ** 31)))
        r = lambda *s: torch.randn(*s, generator=self._gen, device=dev, dtype=torch.float32)
        return r(B, self.act_dim), r(B, self.act_dim), r(B), r(B)

    def _mean_std_buffer(self, dev) -> torch.Tensor:
        if self._mean_std_dev is None or self._mean_std_dev.device != dev:
            self._mean_std_dev = torch.tensor([0.0 if m is None else m for m in self._mean_std], dtype=torch.float32,
                                              device=dev)
        return self._mean_std_dev

    def __compute_gradient(self, data: dict, iteration: int) -> dict:
        start_time = time.time()
        dev = self._device()
        nets, L, P = self.networks, _lib.lib(), _lib.ptr
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        obs, act, rew, obs2, done = (f32(data[k]) for k in ("obs", "act", "rew", "obs2", "done"))
        B, A, O = obs.shape[0], self.act_dim, self.obs_dim
        act = act.reshape(B, A)
        b = self._buffers(B, dev)
        eps_new, eps_next, z1_next, z2_next = self._noise(B, dev)
        alpha = self.__get_alpha()
        pol, polT = nets.policy, nets.policy_target
        n_pol = pol.layerwise(B, 1, "train")
        n_polT = polT.layerwise(B, 1, "infer")
        n_q = layerwise_pair(nets.q1, nets.q2, B, 2, "train")
        n_qT = layerwise_pair(nets.q1_target, nets.q2_target, B, 1, "infer")
        for net, mod in ((n_pol, pol), (n_polT, polT), (n_q.a, nets.q1), (n_q.b, nets.q2), (n_qT.a, nets.q1_target),
                         (n_qT.b, nets.q2_target)):
            net.pack(mod.flat_params.sync())
        mean_std = self._mean_std_buffer(dev)
        unset = int(self._mean_std[0] is None) | (int(self._mean_std[1] is None) << 1)
        st = _lib.stream_ptr
        with torch.cuda.device(dev):
            # new action for the actor loss, next action for the critic target
            n_pol.forward(obs, slot=0, train=True, out=b["logits"])
            _lib.check(L.gops_b200_dsac_sample(P(b["logits"]), P(eps_new), B, A, float(pol.min_log_std),
                                               float(pol.max_log_std), P(b["half"]), P(b["mid"]), P(b["act_new"]),
                                               P(b["logp_new"]), P(obs), O, P(b["qin_new"]), O + A, P(b["stats"]), st()))
            n_polT.forward(obs2, train=False, out=b["logits2"])
            _lib.check(L.gops_b200_dsac_sample(P(b["logits2"]), P(eps_next), B, A, float(polT.min_log_std),
                                               float(polT.max_log_std), P(b["half"]), P(b["mid"]), P(b["act2"]),
                                               P(b["logp2"]), P(obs2), O, P(b["qin2"]), O + A, None, st()))
            # critics: twin loss on (obs, act) against the targets' TD samples at (obs2, act2)
            b["qin"][:, :O].copy_(obs)
            b["qin"][:, O:].copy_(act)
            n_q.forward(b["qin"], slot=0, train=True, out_a=b["q1_out"], out_b=b["q2_out"])
            n_qT.forward(b["qin2"], train=False, out_a=b["t1_out"], out_b=b["t2_out"])
            _lib.check(L.gops_b200_dsact_q_loss(P(b["q1_out"]), P(b["q2_out"]), P(b["t1_out"]), P(b["t2_out"]), P(z1_next),
                                                P(z2_next), P(b["logp2"]), P(rew), P(done), B, float(self.gamma),
                                                float(alpha), float(self.tau_b), P(mean_std), unset, P(b["dq1"]),
                                                P(b["dq2"]), P(b["out"]), st()))
            grads = []
            for q in (nets.q1, nets.q2):
                q.flat_params.bind_grads()
                grads.append(q.flat_params.gbuf[:q.flat_params.gbuf.numel() - 4])
            n_q.backward(b["dq1"], b["dq2"], slot=0, grad_a=grads[0], grad_b=grads[1])
            # actor: alpha logp - min(q1, q2)(obs, new_act), back through the (frozen) critics into the policy
            n_q.forward(b["qin_new"], slot=1, train=True, out_a=b["qn1_out"], out_b=b["qn2_out"])
            _lib.check(L.gops_b200_dsact_policy_loss(P(b["qn1_out"]), P(b["qn2_out"]), P(b["logp_new"]), B, float(alpha),
                                                     float(self.target_entropy), P(b["dqn1"]), P(b["dqn2"]),
                                                     P(b["out"][9:]), P(b["stats"]), st()))
            dx1, dx2 = n_q.backward(b["dqn1"], b["dqn2"], slot=1, want_dx=True)
            _lib.check(L.gops_b200_dsact_sample_backward(P(b["logits"]), P(eps_new), B, A, float(pol.min_log_std),
                                                         float(pol.max_log_std), P(b["half"]), P(dx1), P(dx2), O + A, O,
                                                         float(alpha) / B, P(b["dlogits"]), st()))
            pol.flat_params.bind_grads()
            npol = pol.flat_params.gbuf.numel() - 4
            n_pol.backward(b["dlogits"], slot=0, grad=pol.flat_params.gbuf[:npol])
            b["host"].copy_(b["out"], non_blocking=True)
            torch.cuda.current_stream().synchronize()
        # [loss_q, q1, q2, std1, std2, min std1, min std2, mean_std1, mean_std2,
        #  loss_policy, entropy, mean(logp + H_target), pol mean, pol std]
        h = b["host"].tolist()
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
            tb_tags["alg_time"]: (time.time() - start_time) * 1000,
        }

    def __update(self, iteration: int):
        nets = self.networks
        nets.q1_optimizer.step()
        nets.q2_optimizer.step()
        if iteration % self.delay_update == 0:
            nets.policy_optimizer.step()
            if self.auto_alpha:
                nets.alpha_optimizer.step()
            polyak_update(nets.q1_target.flat_params, nets.q1.flat_params, self.tau)
            polyak_update(nets.q2_target.flat_params, nets.q2.flat_params, self.tau)
            polyak_update(nets.policy_target.flat_params, nets.policy.flat_params, self.tau)
