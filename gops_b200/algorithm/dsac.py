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

import math
import time
from copy import deepcopy
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from gops_b200 import _lib
from gops_b200.algorithm.base import AlgorithmBase, ApprBase
from gops_b200.create_pkg.create_apprfunc import create_apprfunc
from gops_b200.utils.common_utils import get_apprfunc_dict
from gops_b200.utils.flat_params import FusedAdam, ScalarAdam, polyak_update
from gops_b200.utils.tensorboard_setup import tb_tags


class ApproxContainer(ApprBase):
    """One stochastic policy, one distributional action value, their Polyak targets and the temperature."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        q_args = get_apprfunc_dict("value", **kwargs)
        self.q = create_apprfunc(**q_args)
        self.q_target = deepcopy(self.q)
        policy_args = get_apprfunc_dict("policy", **kwargs)
        self.policy = create_apprfunc(**policy_args)
        self.policy_target = deepcopy(self.policy)
        for net in (self.q_target, self.policy_target):
            net.__dict__["_flat_params"] = type(self.q.flat_params)(getattr(net, net._attr))
            net.__dict__["_nets"] = {}
            for p in net.parameters():
                p.requires_grad = False
        self.log_alpha = nn.Parameter(torch.tensor(1, dtype=torch.float32))
        self.q_optimizer = FusedAdam(self.q.flat_params, lr=kwargs["value_learning_rate"])
        self.policy_optimizer = FusedAdam(self.policy.flat_params, lr=kwargs["policy_learning_rate"])
        # the temperature is ONE scalar: torch.optim.Adam's arithmetic on it runs on the host in fp32 (ScalarAdam)
        self.alpha_optimizer = ScalarAdam(self.log_alpha, lr=kwargs["alpha_learning_rate"])
        self.optimizer_dict = {"q": self.q_optimizer, "policy": self.policy_optimizer}
        self.scheduler_dict = {}

    def create_action_distributions(self, logits):
        return self.policy.get_act_dist(logits)


class DSAC(AlgorithmBase):
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
        self.obs_dim, self.act_dim = kwargs["obsv_dim"], kwargs["action_dim"]
        self.noise_override: Optional[Dict[str, torch.Tensor]] = None
        self._gen = None
        self._buf = {}
        if torch.cuda.is_available():
            self.networks.cuda()

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "auto_alpha", "alpha", "bound", "delay_update")

    # ------------------------------------------------------------------------------------------------ plugin surface
    def local_update(self, data: dict, iteration: int) -> dict:
        tb_info = self.__compute_gradient(data, iteration)
        self.__update(iteration)
        return tb_info

    def get_remote_update_info(self, data: dict, iteration: int) -> Tuple[dict, dict]:
        tb_info = self.__compute_gradient(data, iteration)
        update_info = {"q_grad": [p._grad for p in self.networks.q.parameters()],
                       "policy_grad": [p._grad for p in self.networks.policy.parameters()], "iteration": iteration}
        if self.auto_alpha:
            update_info["log_alpha_grad"] = self.networks.alpha_optimizer.grad
        return tb_info, update_info

    def remote_update(self, update_info: dict):
        for p, grad in zip(self.networks.q.parameters(), update_info["q_grad"]):
            p._grad = grad
        for p, grad in zip(self.networks.policy.parameters(), update_info["policy_grad"]):
            p._grad = grad
        if self.auto_alpha:
            self.networks.alpha_optimizer.grad = update_info["log_alpha_grad"]
        self.__update(update_info["iteration"])

    # ------------------------------------------------------------------------------------------------ internals
    def _device(self) -> torch.device:
        p = next(self.networks.q.parameters())
        if not p.is_cuda:
            if not torch.cuda.is_available():
                raise RuntimeError("gops_b200: no CUDA device -- the DSAC update has no CPU fallback")
            self.networks.cuda()
            p = next(self.networks.q.parameters())
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
                                 q_out=z(B, 2), q2_out=z(B, 2), qn_out=z(B, 2), dq=z(B, 2), dqn=z(B, 2),
                                 dlogits=z(B, 2 * A), stats=z(2 * B), out=z(8).contiguous(),
                                 host=torch.zeros(8).pin_memory())
            pol = self.networks.policy
            b["half"] = ((pol.act_high_lim - pol.act_low_lim) / 2).to(dev, torch.float32).contiguous()
            b["mid"] = ((pol.act_high_lim + pol.act_low_lim) / 2).to(dev, torch.float32).contiguous()
        return b

    def _noise(self, B: int, dev):
        if self.noise_override is not None:
            n = self.noise_override
            return (n["eps_new"].to(dev, torch.float32).reshape(B, self.act_dim).contiguous(),
                    n["eps_next"].to(dev, torch.float32).reshape(B, self.act_dim).contiguous(),
                    n["z_next"].to(dev, torch.float32).reshape(B).contiguous())
        if self._gen is None or self._gen.device != dev:
            self._gen = torch.Generator(device=dev).manual_seed(int(torch.initial_seed() % (2 ** 31)))
        r = lambda *s: torch.randn(*s, generator=self._gen, device=dev, dtype=torch.float32)
        return r(B, self.act_dim), r(B, self.act_dim), r(B)

    def __compute_gradient(self, data: dict, iteration: int) -> dict:
        start_time = time.time()
        dev = self._device()
        nets, L = self.networks, _lib.lib()
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        obs, act, rew, obs2, done = (f32(data[k]) for k in ("obs", "act", "rew", "obs2", "done"))
        B, A, O = obs.shape[0], self.act_dim, self.obs_dim
        act = act.reshape(B, A)
        b = self._buffers(B, dev)
        eps_new, eps_next, z_next = self._noise(B, dev)
        alpha = self.__get_alpha()
        pol, polT, q, qT = nets.policy, nets.policy_target, nets.q, nets.q_target
        n_pol = pol.layerwise(B, 1, "train")
        n_polT = polT.layerwise(B, 1, "infer")
        n_q = q.layerwise(B, 2, "train")
        n_qT = qT.layerwise(B, 1, "infer")
        for net, mod in ((n_pol, pol), (n_polT, polT), (n_q, q), (n_qT, qT)):
            net.pack(mod.flat_params.sync())
        st = _lib.stream_ptr
        with torch.cuda.device(dev):
            # new action for the actor loss, next action for the critic target
            n_pol.forward(obs, slot=0, train=True, out=b["logits"])
            _lib.check(L.gops_b200_dsac_sample(_lib.ptr(b["logits"]), _lib.ptr(eps_new), B, A, float(pol.min_log_std),
                                               float(pol.max_log_std), _lib.ptr(b["half"]), _lib.ptr(b["mid"]),
                                               _lib.ptr(b["act_new"]), _lib.ptr(b["logp_new"]), _lib.ptr(obs), O,
                                               _lib.ptr(b["qin_new"]), O + A, _lib.ptr(b["stats"]), st()))
            n_polT.forward(obs2, train=False, out=b["logits2"])
            _lib.check(L.gops_b200_dsac_sample(_lib.ptr(b["logits2"]), _lib.ptr(eps_next), B, A, float(polT.min_log_std),
                                               float(polT.max_log_std), _lib.ptr(b["half"]), _lib.ptr(b["mid"]),
                                               _lib.ptr(b["act2"]), _lib.ptr(b["logp2"]), _lib.ptr(obs2), O,
                                               _lib.ptr(b["qin2"]), O + A, None, st()))
            # critic: loss on (obs, act) against the clipped TD target from q_target(obs2, act2)
            b["qin"][:, :O].copy_(obs)
            b["qin"][:, O:].copy_(act)
            n_q.forward(b["qin"], slot=0, train=True, out=b["q_out"])
            n_qT.forward(b["qin2"], train=False, out=b["q2_out"])
            _lib.check(L.gops_b200_dsac_q_loss(_lib.ptr(b["q_out"]), _lib.ptr(b["q2_out"]), _lib.ptr(z_next),
                                               _lib.ptr(b["logp2"]), _lib.ptr(rew), _lib.ptr(done), B, float(self.gamma),
                                               float(alpha), int(bool(self.bound)), _lib.ptr(b["dq"]), _lib.ptr(b["out"]), st()))
            q.flat_params.bind_grads()
            nq = q.flat_params.gbuf.numel() - 4
            n_q.backward(b["dq"], slot=0, grad=q.flat_params.gbuf[:nq])
            # actor: alpha logp - q(obs, new_act), back through the (frozen) critic into the policy
            n_q.forward(b["qin_new"], slot=1, train=True, out=b["qn_out"])
            _lib.check(L.gops_b200_dsac_policy_loss(_lib.ptr(b["qn_out"]), _lib.ptr(b["logp_new"]), B, float(alpha),
                                                    float(self.target_entropy), _lib.ptr(b["dqn"]),
                                                    C_ptr_off(b["out"], 3), _lib.ptr(b["stats"]), st()))
            d_qin = n_q.backward(b["dqn"], slot=1, grad=None, want_dx=True)
            _lib.check(L.gops_b200_dsac_sample_backward(_lib.ptr(b["logits"]), _lib.ptr(eps_new), B, A,
                                                        float(pol.min_log_std), float(pol.max_log_std), _lib.ptr(b["half"]),
                                                        _lib.ptr(d_qin), O + A, O, float(alpha) / B, _lib.ptr(b["dlogits"]), st()))
            pol.flat_params.bind_grads()
            npol = pol.flat_params.gbuf.numel() - 4
            n_pol.backward(b["dlogits"], slot=0, grad=pol.flat_params.gbuf[:npol])
            b["host"].copy_(b["out"], non_blocking=True)
            torch.cuda.current_stream().synchronize()
        h = b["host"].tolist()      # [loss_q, mean q, mean q_std, loss_policy, entropy, mean(logp + H_target), pol mean, pol std]
        if self.auto_alpha:         # loss_alpha = -log_alpha * mean(logp + target_entropy)   (dsac.py:272-278)
            self.networks.alpha_optimizer.grad = -h[5]
        return {
            "DSAC/critic_avg_q-RL iter": h[1], "DSAC/critic_avg_std-RL iter": h[2],
            tb_tags["loss_actor"]: h[3], "DSAC/policy_mean-RL iter": h[6], "DSAC/policy_std-RL iter": h[7],
            "DSAC/entropy-RL iter": h[4], "DSAC/alpha-RL iter": alpha,
            tb_tags["loss_critic"]: h[0],
            tb_tags["alg_time"]: (time.time() - start_time) * 1000,
        }

    def __update(self, iteration: int):
        nets = self.networks
        nets.q_optimizer.step()
        if iteration % self.delay_update == 0:
            nets.policy_optimizer.step()
            if self.auto_alpha:
                nets.alpha_optimizer.step()
            polyak_update(nets.q_target.flat_params, nets.q.flat_params, self.tau)
            polyak_update(nets.policy_target.flat_params, nets.policy.flat_params, self.tau)


def C_ptr_off(t: torch.Tensor, offset: int):
    import ctypes as C
    return C.c_void_p(t.data_ptr() + 4 * offset)
