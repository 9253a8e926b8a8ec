"""Relaxed Policy Iteration (RPI), H100 edition.

Same plugin surface as the reference (gops/algorithm/rpi.py: ApproxContainer :37-108, RPI :111-327) for its MLP example
on pyth_oscillatorconti: a StateValue V learns the continuous-time zero-sum (H-infinity) value by driving the HJI
Hamiltonian H = c(x, u, w) + dV/dx . f(x, u, w) to zero, with the control u = -0.5 x0 dV/dx1 and the worst disturbance
w = 0.5 / gamma_atte^2 x1 dV/dx1 in closed form from the target value's gradient.

Every Newton iteration (`local_update`) is ONE launch of gops_b200_rpi_newton (csrc/rpi.cu), a thread-block cluster of
B / 64 CTAs that runs the reference's whole policy-evaluation loop on the device: sample, Hamiltonian loss and gradient,
cluster reduction, Adam, the Hamiltonian norm on the iteration's fixed state set and the stopping test
|H_after| > 0.88 |H_before|, then value_target <- value.  The host reads four numbers per iteration.

The reference's sampler, reproduced as it behaves (see DESIGN.md, "RPI"): the raw action and disturbance drive the
unwrapped model (no ScaleAction / clipping), every inner step draws a fresh reset state that done or truncated samples
take, and the model's step counter is never reset, so a sample is truncated on every step once the total number of
inner steps exceeds its max_step_per_episode.  The loss itself goes through the wrapped model (u = 5 clip(a),
w = clip(w) / gamma_atte).

Reset draws are made with torch on the device before each launch ([1 + max_step_update_value][B][2], U[-r, r] per
component, from a generator seeded with `seed`): row 0 is the iteration's set_state, row n the draw of inner step n.
`reset_override` replaces them with given draws; `obs`, `max_step_per_episode` and `step_per_episode` are the sampler
state and may be assigned."""
__all__ = ["ApproxContainer", "RPI"]

import time
from copy import deepcopy
from typing import Any, Optional

import numpy as np
import torch
import torch.nn as nn

from gops_b200 import _lib
from gops_b200.algorithm.base import AlgorithmBase, ApprBase
from gops_b200.create_pkg.create_apprfunc import create_apprfunc
from gops_b200.create_pkg.create_env_model import create_env_model
from gops_b200.utils.common_utils import get_apprfunc_dict
from gops_b200.utils.flat_params import FusedAdam
from gops_b200.utils.tensorboard_setup import tb_tags

TILE, MAX_BATCH = 64, 512
ACTIVATIONS = ("relu", "elu", "gelu", "selu", "sigmoid", "tanh")


def check_config(**kwargs):
    """The configurations the RPI kernels run, refused before anything is built or launched."""
    if kwargs.get("env_id") != "pyth_oscillatorconti":
        raise ValueError("RPI is built for env_id='pyth_oscillatorconti'")
    if not kwargs.get("is_adversary", False):
        raise ValueError("RPI needs is_adversary=True (the reference crashes without an adversary)")
    if kwargs.get("value_func_type") != "MLP" or kwargs.get("value_func_name", "StateValue") != "StateValue":
        raise NotImplementedError("RPI on the GPU supports an MLP StateValue only")
    if list(kwargs.get("value_hidden_sizes", [])) != [64, 64]:
        raise NotImplementedError(f"RPI kernels need value_hidden_sizes=[64, 64], got {kwargs.get('value_hidden_sizes')}")
    if kwargs.get("value_hidden_activation") not in ACTIVATIONS:
        raise NotImplementedError(f"RPI kernels support the hidden activations {ACTIVATIONS}")
    if kwargs.get("value_output_activation", "linear") != "linear":
        raise NotImplementedError("RPI kernels support value_output_activation='linear' only")
    B = int(kwargs.get("reset_batch_size", 0))
    if B <= 0 or B % TILE or B > MAX_BATCH:
        raise ValueError(f"RPI needs reset_batch_size a multiple of 64 and at most 512 (one CTA cluster), got {B}")
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        raise NotImplementedError("RPI runs on one GPU (the reference's RPI is serial only)")


class ApproxContainer(ApprBase):
    """value and value_target StateValues (rpi.py:37-103); the target's gradient gives the policy."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        check_config(**kwargs)
        self.gamma_atte = float(kwargs["gamma_atte"])
        self.value = create_apprfunc(**get_apprfunc_dict("value", **kwargs))
        for m in self.value.v:                         # rpi.py:63-71: Xavier-uniform weights, zero biases
            if isinstance(m, nn.Linear):
                fan_out, fan_in = m.weight.shape
                w_bound = np.sqrt(6.0 / (fan_in + fan_out))
                m.weight.data.uniform_(-w_bound, w_bound)
                m.bias.data.fill_(0)
        self.value_target = deepcopy(self.value)

    def action_and_adversary(self, batch_obs: torch.Tensor) -> torch.Tensor:
        """[a, w] = [best_act, worst_adv] from dV_target/dx (raw, unscaled), one kernel launch."""
        flat = self.value_target.flat_params.sync()
        if not flat.is_cuda:
            raise RuntimeError("gops_b200 RPI networks run on a CUDA device only (no CPU fallback); call .cuda()")
        x = batch_obs.detach().to(flat.device, torch.float32).reshape(-1, 2).contiguous()
        out = torch.empty_like(x)
        with torch.cuda.device(flat.device):
            _lib.check(_lib.lib().gops_b200_rpi_policy(
                _lib.ptr(flat), _lib.ACT_IDS[self.value._hidden_act], self.gamma_atte, _lib.ptr(x), x.shape[0],
                _lib.ptr(out), _lib.stream_ptr()))
        return out.to(batch_obs.device)

    def policy(self, batch_obs: torch.Tensor) -> torch.Tensor:
        return self.action_and_adversary(batch_obs)[:, :1]

    @staticmethod
    def create_action_distributions(logits):
        from gops_b200.utils.act_distribution_type import DiracDistribution
        return DiracDistribution(logits)


class RPI(AlgorithmBase):
    """:param int max_newton_iteration: Newton iterations of a run.  :param int max_step_update_value: cap on the inner
    (policy-evaluation) steps of one iteration.  :param float learning_rate: Adam's lr (betas (0.9, 0.99))."""

    def __init__(self, index: int = 0, max_newton_iteration: int = 50, max_step_update_value: int = 10000,
                 print_interval: int = 1, learning_rate: float = 1e-3, **kwargs: Any):
        check_config(**kwargs)
        super().__init__(index, **kwargs)
        self.max_newton_iteration = max_newton_iteration
        self.max_step_update_value = max_step_update_value
        self.print_interval = print_interval
        self.num_update_value = 0
        self.norm_hamiltonian_before = 0
        self.norm_hamiltonian_after = self.max_step_update_value ** 3
        self.grad_step = np.ones([int(self.max_newton_iteration), 1], dtype="float32")
        self.is_adversary = True
        self.env_model = create_env_model(**kwargs)
        model = self.env_model.unwrapped
        self.obsv_dim, self.act_dim = model.state_dim, model.action_dim
        self.batch = model.sample_batch_size
        self.gamma_atte = float(model.gamma_atte)
        self.initial_state_range = [float(r) for r in model.initial_state_range]
        self.state_threshold = [float(t) for t in model.state_threshold]
        # sampler state: the reference's first reset and the model's per-sample episode caps; one step counter
        self.obs = self.env_model.reset()
        self.max_step_per_episode = model.max_step_per_episode.clone()
        self.step_per_episode = 0
        self.networks = ApproxContainer(**kwargs)
        self.learning_rate = learning_rate
        self.approximate_optimizer = FusedAdam(self.networks.value.flat_params, lr=learning_rate, betas=(0.9, 0.99))
        self.seed = int(kwargs.get("seed", 0) or 0)
        self.reset_override: Optional[torch.Tensor] = None
        self.record_trace = False
        self.last_trace: Optional[torch.Tensor] = None

    @property
    def adjustable_parameters(self):
        return ("max_newton_iteration",)

    def _device(self) -> torch.device:
        p = next(self.networks.parameters())
        if not p.is_cuda:
            if not torch.cuda.is_available():
                raise RuntimeError("gops_b200: no CUDA device -- the RPI update has no CPU fallback")
            self.networks.cuda()
        return next(self.networks.parameters()).device

    def _draws(self, dev) -> torch.Tensor:
        """[1 + max_step_update_value][B][2] reset draws of one Newton iteration (or the override)."""
        B = self.batch
        if self.reset_override is not None:
            d = self.reset_override.to(dev, torch.float32).contiguous()
            if d.dim() != 3 or d.shape[0] < 2 or tuple(d.shape[1:]) != (B, 2):
                raise ValueError(f"reset_override must be [1 + steps, {B}, 2], got {tuple(d.shape)}")
            return d
        st = self.__dict__
        if st.get("_gen") is None:
            st["_gen"] = torch.Generator(device=dev).manual_seed(self.seed)
        rows = 1 + int(self.max_step_update_value)
        buf = st.get("_draw_buf")
        if buf is None or buf.shape[0] != rows or buf.device != dev:
            buf = st["_draw_buf"] = torch.empty((rows, B, 2), dtype=torch.float32, device=dev)
        for i in range(2):
            r = self.initial_state_range[i]
            buf[:, :, i].uniform_(-r, r, generator=st["_gen"])
        return buf

    def local_update(self, data_useless, iteration: int) -> dict:
        start_time = time.time()
        dev = self._device()
        nets, opt = self.networks, self.approximate_optimizer
        target = nets.value_target.flat_params.sync()
        flat, m, v, step0, group = opt.multi_step_state()
        draws = self._draws(dev)
        st = self.__dict__
        if st.get("_dev_state") is None or st["_dev_state"][0].device != dev:
            st["_dev_state"] = (torch.empty((self.batch, 2), dtype=torch.float32, device=dev),
                                torch.empty(self.batch, dtype=torch.int32, device=dev),
                                torch.empty(1, dtype=torch.int32, device=dev),
                                torch.zeros(8, dtype=torch.float32, device=dev))
        x, max_step, counter, out = st["_dev_state"]
        x.copy_(torch.as_tensor(self.obs).reshape(self.batch, 2))
        max_step.copy_(torch.as_tensor(self.max_step_per_episode).reshape(-1).to(torch.int32))
        counter.fill_(int(self.step_per_episode))
        max_steps = int(self.max_step_update_value)
        trace = torch.zeros((max_steps, 2), dtype=torch.float32, device=dev) if self.record_trace else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gops_b200_rpi_newton(
                _lib.ptr(flat), _lib.ptr(target), _lib.ptr(m), _lib.ptr(v), int(step0), float(group["lr"]),
                float(group["betas"][0]), float(group["betas"][1]), float(group["eps"]),
                _lib.ACT_IDS[nets.value._hidden_act], self.gamma_atte, self.state_threshold[0], self.state_threshold[1], _lib.ptr(x), _lib.ptr(max_step),
                _lib.ptr(counter), _lib.ptr(draws), int(draws.shape[0]), max_steps, self.batch, _lib.ptr(out),
                _lib.ptr(trace), _lib.stream_ptr()))
        host = out.cpu().tolist()          # the iteration's one host read
        n = int(host[0])
        if host[4] and n < max_steps:
            raise ValueError(f"reset_override holds draws for {draws.shape[0] - 1} inner steps, the iteration needed more")
        opt.advance(n)
        self.obs = x.clone()
        self.step_per_episode = int(self.step_per_episode) + n
        self.num_update_value = n
        self.norm_hamiltonian_before, self.norm_hamiltonian_after = host[2], host[3]
        self.last_trace = trace[:n].clone() if trace is not None else None
        grad_info = {"iteration": iteration, "num_update_value": n, tb_tags["loss_critic"]: host[1],
                     tb_tags["alg_time"]: (time.time() - start_time) * 1000}
        if iteration % self.print_interval == 0:
            if iteration < len(self.grad_step):
                self.grad_step[iteration, 0] = n
            print(f"Newton ite: {iteration}, grad step = {n:d}")
        return grad_info

    def loss_and_grad(self, obs: torch.Tensor, act_adv: torch.Tensor):
        """One Hamiltonian loss mean|c + dV/dx . f| of the wrapped model at (obs, raw [a, w]) and its gradient, which is
        written to the value's flat gradient (p.grad views), as `loss.backward()` in RPI.__compute_loss (rpi.py:218-229)."""
        dev = self._device()
        fp = self.networks.value.flat_params
        flat = fp.sync()
        fp.bind_grads()
        x = obs.detach().to(dev, torch.float32).reshape(-1, 2).contiguous()
        a = act_adv.detach().to(dev, torch.float32).reshape(-1, 2).contiguous()
        B = x.shape[0]
        if B % TILE:
            raise ValueError(f"loss_and_grad needs a batch that is a multiple of 64, got {B}")
        lib = _lib.lib()
        scratch = torch.empty(int(lib.gops_b200_rpi_scratch_floats(B)), dtype=torch.float32, device=dev)
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.gops_b200_rpi_loss_grad(
                _lib.ptr(flat), _lib.ACT_IDS[self.networks.value._hidden_act], self.gamma_atte, _lib.ptr(x), _lib.ptr(a),
                B, _lib.ptr(scratch), _lib.ptr(fp.gbuf), _lib.ptr(loss), _lib.stream_ptr()))
        return loss
