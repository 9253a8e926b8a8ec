"""Host plumbing shared by the soft actor-critic family: DSAC, DSAC-T and SAC.

One update samples the new action at obs and the next action at obs2 (tanh-Gaussian reparameterisation, csrc/dsac.cu),
builds the [obs | act] critic input, runs the algorithm's critic and actor losses (`_losses`: its critics' passes and
loss kernels, ending in the policy's output gradient `dlogits`), back-propagates the policy, and reads the update's
scalars back once.  Then the critics take an Adam step on every update; the policy, the temperature and the Polyak
averages of the targets every `delay_update` updates."""
import time
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from gops_b200 import _lib
from gops_b200.algorithm.base import AlgorithmBase
from gops_b200.ops.layerwise_mlp import layerwise_pair
from gops_b200.utils.flat_params import GRAD_TAIL, polyak_update
from gops_b200.utils.tensorboard_setup import tb_tags


class SoftActorCritic(AlgorithmBase):
    _critics: Tuple[str, ...]                    # the trained critics; one, or twins run as paired passes
    _policy_target: bool                         # next action from policy_target, or from slot 1 of the policy's handle
    _noise_shapes: Tuple[Tuple[str, str], ...]   # (name, "BA": [B, act_dim] | "B": [B]) in the order of the draws
    _n_out: int                                  # floats of the update's scalar read-back

    def _init_soft_ac(self, kwargs):
        self.obs_dim, self.act_dim = kwargs["obsv_dim"], kwargs["action_dim"]
        self.noise_override: Optional[Dict[str, torch.Tensor]] = None
        self._gen = None
        self._buf = {}
        if torch.cuda.is_available():
            self.networks.cuda()

    # ------------------------------------------------------------------------------------------------ plugin surface
    def local_update(self, data: dict, iteration: int) -> dict:
        tb_info = self._compute_gradient(data)
        self._update(iteration)
        return tb_info

    def get_remote_update_info(self, data: dict, iteration: int) -> Tuple[dict, dict]:
        tb_info = self._compute_gradient(data)
        update_info = {key: [p._grad for p in mod.parameters()] for key, mod in self._trained()}
        update_info["iteration"] = iteration
        if self.auto_alpha:
            update_info["log_alpha_grad"] = self.networks.alpha_optimizer.grad
        return tb_info, update_info

    def remote_update(self, update_info: dict):
        for key, mod in self._trained():
            for p, grad in zip(mod.parameters(), update_info[key]):
                p._grad = grad
        if self.auto_alpha:
            self.networks.alpha_optimizer.grad = update_info["log_alpha_grad"]
        self._update(update_info["iteration"])

    # ------------------------------------------------------------------------------------------------ internals
    def _trained(self):
        """(grad key, module) of every network the optimizers step."""
        return [(f"{name}_grad", getattr(self.networks, name)) for name in self._critics + ("policy",)]

    def _alpha(self) -> float:
        return float(np.exp(np.float32(self.networks.log_alpha.item()))) if self.auto_alpha else self.alpha

    def _buffers(self, B: int, dev) -> dict:
        b = self._buf
        if b.get("B") != B or b.get("dev") != dev:
            A, O = self.act_dim, self.obs_dim
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
            b = self._buf = dict(B=B, dev=dev, logits=z(B, 2 * A), logits2=z(B, 2 * A), act_new=z(B, A), act2=z(B, A),
                                 logp_new=z(B), logp2=z(B), qin=z(B, O + A), qin_new=z(B, O + A), qin2=z(B, O + A),
                                 dlogits=z(B, 2 * A), out=z(self._n_out), host=torch.zeros(self._n_out).pin_memory(),
                                 **self._critic_buffers(B, z))
            pol = self.networks.policy
            b["half"] = ((pol.act_high_lim - pol.act_low_lim) / 2).to(dev, torch.float32).contiguous()
            b["mid"] = ((pol.act_high_lim + pol.act_low_lim) / 2).to(dev, torch.float32).contiguous()
        return b

    def _noise(self, B: int, dev) -> Dict[str, torch.Tensor]:
        shapes = [(name, (B, self.act_dim) if shape == "BA" else (B,)) for name, shape in self._noise_shapes]
        if self.noise_override is not None:
            n = self.noise_override
            return {name: n[name].to(dev, torch.float32).reshape(shape).contiguous() for name, shape in shapes}
        if self._gen is None or self._gen.device != dev:
            self._gen = torch.Generator(device=dev).manual_seed(int(torch.initial_seed() % (2 ** 31)))
        r = lambda shape: torch.randn(shape, generator=self._gen, device=dev, dtype=torch.float32)
        return {name: r(shape) for name, shape in shapes}

    @staticmethod
    def _grad_view(net) -> torch.Tensor:
        """Points the net's p.grad at its flat gradient buffer; returns that buffer without its scalar tail."""
        net.flat_params.bind_grads()
        return net.flat_params.gbuf[:-GRAD_TAIL]

    def _critic_handles(self, B: int):
        """Library handles of the critics (training, 2 slots) and their targets, packed with the current weights after
        the policy's."""
        nets = self.networks
        crit = [getattr(nets, name) for name in self._critics]
        targ = [getattr(nets, name + "_target") for name in self._critics]
        if len(crit) == 2:
            n_q, n_qT = layerwise_pair(*crit, B, 2, "train"), layerwise_pair(*targ, B, 1, "infer")
            return n_q, n_qT, [(n_q.a, crit[0]), (n_q.b, crit[1]), (n_qT.a, targ[0]), (n_qT.b, targ[1])]
        n_q, n_qT = crit[0].layerwise(B, 2, "train"), targ[0].layerwise(B, 1, "infer")
        return n_q, n_qT, [(n_q, crit[0]), (n_qT, targ[0])]

    def _compute_gradient(self, data: dict) -> dict:
        start_time = time.time()
        dev = self._device()
        nets, L, P, st = self.networks, _lib.lib(), _lib.ptr, _lib.stream_ptr
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        obs, act, rew, obs2, done = (f32(data[k]) for k in ("obs", "act", "rew", "obs2", "done"))
        B, A, O = obs.shape[0], self.act_dim, self.obs_dim
        act = act.reshape(B, A)
        b = self._buffers(B, dev)
        noise = self._noise(B, dev)
        alpha = self._alpha()
        pol = nets.policy
        if self._policy_target:
            pol_next, next_slot = nets.policy_target, 0
            n_pol, n_next = pol.layerwise(B, 1, "train"), pol_next.layerwise(B, 1, "infer")
            packs = [(n_pol, pol), (n_next, pol_next)]
        else:                                   # slot 0: obs (trained), slot 1: obs2 (next action)
            pol_next, next_slot = pol, 1
            n_pol = n_next = pol.layerwise(B, 2, "train")
            packs = [(n_pol, pol)]
        n_q, n_qT, critic_packs = self._critic_handles(B)
        for net, mod in packs + critic_packs:
            net.pack(mod.flat_params.sync())
        with torch.cuda.device(dev):
            # new action for the actor loss (with the policy's mean / std statistics where the loss reports them), next
            # action for the critic target
            n_pol.forward(obs, slot=0, train=True, out=b["logits"])
            _lib.check(L.gops_b200_dsac_sample(P(b["logits"]), P(noise["eps_new"]), B, A, float(pol.min_log_std),
                                               float(pol.max_log_std), P(b["half"]), P(b["mid"]), P(b["act_new"]),
                                               P(b["logp_new"]), P(obs), O, P(b["qin_new"]), O + A, P(b.get("stats")),
                                               st()))
            n_next.forward(obs2, slot=next_slot, train=False, out=b["logits2"])
            _lib.check(L.gops_b200_dsac_sample(P(b["logits2"]), P(noise["eps_next"]), B, A, float(pol_next.min_log_std),
                                               float(pol_next.max_log_std), P(b["half"]), P(b["mid"]), P(b["act2"]),
                                               P(b["logp2"]), P(obs2), O, P(b["qin2"]), O + A, None, st()))
            b["qin"][:, :O].copy_(obs)
            b["qin"][:, O:].copy_(act)
            self._losses(b, n_q, n_qT, rew, done, noise, alpha)
            n_pol.backward(b["dlogits"], slot=0, grad=self._grad_view(pol))
            b["host"].copy_(b["out"], non_blocking=True)
            torch.cuda.current_stream().synchronize()
        tb_info = self._tb(b["host"].tolist(), alpha)
        tb_info[tb_tags["alg_time"]] = (time.time() - start_time) * 1000
        return tb_info

    def _update(self, iteration: int):
        nets = self.networks
        for name in self._critics:
            nets.optimizer_dict[name].step()
        if iteration % self.delay_update == 0:
            nets.policy_optimizer.step()
            if self.auto_alpha:
                nets.alpha_optimizer.step()
            for name in self._critics:
                polyak_update(getattr(nets, name + "_target").flat_params, getattr(nets, name).flat_params, self.tau)
            if self._policy_target:
                polyak_update(nets.policy_target.flat_params, nets.policy.flat_params, self.tau)

    # ------------------------------------------------------------------------------------------------ per algorithm
    def _critic_buffers(self, B: int, z) -> dict:
        """The critics' outputs and output gradients (`z(*shape)` allocates zeros on the device)."""
        raise NotImplementedError

    def _losses(self, b: dict, n_q, n_qT, rew: torch.Tensor, done: torch.Tensor, noise: Dict[str, torch.Tensor],
                alpha: float):
        """Critic and actor losses into b["out"], the critics' weight gradients, the policy's output gradient into
        b["dlogits"]."""
        raise NotImplementedError

    def _tb(self, h: list, alpha: float) -> dict:
        """The tb values of the read-back scalars `h` (the temperature gradient is set from them here)."""
        raise NotImplementedError
