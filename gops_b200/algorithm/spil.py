"""Separated Proportional-Integral Lagrangian (SPIL), H100 edition.

Same plugin surface as the reference (gops/algorithm/spil.py: ApproxContainer :32-70, SPIL :73-270): chance-constrained
model-based RL on pyth_veh3dofconti_errcstr (two constraints of the incoming observation) and pyth_mobilerobot (one
obstacle-distance constraint of the raw next state, with obstacle noise).  Every update runs both passes of the reference's `__compute_gradient`
(:160-180), each as ONE fused CUDA kernel (csrc/kernel.cuh, constraint mode 4):

  value pass   INFADP's PEV rollout (:182-212) without the (~d) mask on the terminal v_target, counting per constraint the
               trajectories that stayed safe (constraint <= 0 on every step);
  controller   `__spil_get_weight` (:257-270) as one device kernel in float64 that turns the batch's safe probability
               into the weights [w_r, w_c0, w_c1] -- no host round trip;
  policy pass  FHADP's differentiated rollout with the DetermPolicy (:214-255): -mean(w_r R + sum_i w_c,i prod_k Phi(c_k,i)),
               the weights read from device memory;

then both fused Adam steps and both Polyak averages (:146-158).  With several GPUs the value pass's safe counts are
summed by the gradient exchange, so every rank runs the controller on the GLOBAL safe probability and the replicas keep
identical multipliers (the reference's Ray replicas each run a controller of their own).

pyth_mobilerobot's obstacle noise is drawn on the device once per pass ([forward_step][B][2], the env model's
generator), or taken from `noise_override` = {"value": ..., "policy": ...}.  With one constraint the controller runs
with chance_thre1 = 0 on a zero safe count: lam_1 = 0 exactly, so the weights equal the reference's 1 / (1 + lam.sum())
and lam / (1 + lam.sum())."""
__all__ = ["SPIL"]

import time
from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch

from gops_b200 import _lib
from gops_b200.algorithm.base import AlgorithmBase, FusedADPMixin
from gops_b200.algorithm.infadp import ApproxContainer   # noqa: F401  (ApproxContainer: registry contract)
from gops_b200.create_pkg.create_env_model import create_env_model
from gops_b200.utils.flat_params import GRAD_TAIL, polyak_update
from gops_b200.utils.tensorboard_setup import tb_tags

MODE_SPIL = 4        # gops_b200_plan_set_constraint mode
CONSTRAINT_DIM = {"pyth_veh3dofconti_errcstr": 2, "pyth_mobilerobot": 1}     # the fused kernel's constraint providers


class SPIL(AlgorithmBase, FusedADPMixin):
    """:param float gamma: discount factor.  :param float tau: Polyak coefficient of both targets.
    :param int forward_step: model rollout length of both passes.  `pev_step` / `pim_step` are stored but unused, as in
    the reference: both networks are updated on every iteration."""

    def __init__(self, index: int = 0, gamma: float = 0.99, tau: float = 0.005, pev_step: int = 1, pim_step: int = 1,
                 forward_step: int = 25, **kwargs: Any):
        env_id = kwargs.get("env_id")
        if env_id not in CONSTRAINT_DIM:
            raise ValueError("SPIL is built for env_id='pyth_veh3dofconti_errcstr' and 'pyth_mobilerobot' (the fused "
                             "kernel's constraint providers)")
        if kwargs.get("constraint_dim") != CONSTRAINT_DIM[env_id]:
            raise ValueError(f"SPIL on {env_id} needs constraint_dim={CONSTRAINT_DIM[env_id]}"
                             + (" (|y_err| and |u_err| constraints)" if env_id == "pyth_veh3dofconti_errcstr" else
                                " (one obstacle-distance constraint)"))
        if env_id == "pyth_mobilerobot" and (kwargs.get("repeat_num") or 1) > 1:
            raise ValueError("SPIL on pyth_mobilerobot: repeat_num > 1 is not supported (one noise draw per model step)")
        super().__init__(index, **kwargs)
        self.networks = ApproxContainer(**kwargs)
        self.envmodel = create_env_model(**kwargs)
        self.gamma = gamma
        self.tau = tau
        self.pev_step = pev_step
        self.pim_step = pim_step
        self.forward_step = forward_step
        self.reward_scale = 1.0        # hard-coded as in the reference; the reward_scale kwarg reaches ShapingReward only
        self.n_constraint = kwargs["constraint_dim"]
        self.Kp = 60
        self.Ki = 0.02
        self.Kd = 0
        self.chance_thre = np.array([0.97] * self.n_constraint)
        self.noisy = env_id == "pyth_mobilerobot"
        self.noise_override: Optional[Dict[str, torch.Tensor]] = None
        self.tb_info = dict()
        self._init_fused()

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "pev_step", "pim_step", "forward_step", "reward_scale")

    # ---- controller state (lives on the device) --------------------------------------------------------------------
    def _ctl(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """float64 [delta_i(2), safe_prob_pre(2), lam(2)] and the policy pass's float32 weights [w_r, w_c0, w_c1]."""
        if "_spil_state" not in self.__dict__:
            dev = self._device()
            self._spil_state = torch.zeros(6, dtype=torch.float64, device=dev)
            self._spil_w = torch.zeros(3, dtype=torch.float32, device=dev)
        return self._spil_state, self._spil_w

    @property
    def delta_i(self) -> np.ndarray:
        return self._ctl()[0][0:self.n_constraint].cpu().numpy()

    @delta_i.setter
    def delta_i(self, value):
        st = self._ctl()[0]
        st[0:self.n_constraint] = torch.as_tensor(np.asarray(value, dtype=np.float64), device=st.device)

    @property
    def safe_prob(self) -> np.ndarray:
        """safe probability of the most recent value pass (float32, as the reference's traj_issafe.mean(0))."""
        return self._ctl()[0][2:2 + self.n_constraint].cpu().numpy().astype(np.float32)

    @property
    def lam(self) -> np.ndarray:
        return self._ctl()[0][4:4 + self.n_constraint].cpu().numpy()

    # ---- update ------------------------------------------------------------------------------------------------------
    def local_update(self, data: dict, iteration: int) -> dict:
        start_time = time.time()
        nets = self.networks
        tail_v = self._launch_and_step(lambda: self._value_pass(data), nets.v_optimizer)
        self._controller(tail_v, data)
        tail_p = self._launch_and_step(lambda: self._policy_pass(data), nets.policy_optimizer)
        self._polyak()
        self._publish(tail_v, tail_p, start_time)
        return self.tb_info

    def get_remote_update_info(self, data: dict, iteration: int) -> Tuple[dict, dict]:
        start_time = time.time()
        tail_v = self._value_pass(data)
        self._controller(tail_v, data)
        tail_p = self._policy_pass(data)
        self._publish(tail_v, tail_p, start_time)
        update_info = {name: [p.grad for p in self.networks.net_dict[name].parameters()] for name in ("v", "policy")}
        return self.tb_info, update_info

    def remote_update(self, update_info: dict):
        for net_name, grads in update_info.items():
            for p, grad in zip(self.networks.net_dict[net_name].parameters(), grads):
                p.grad = grad
        for net_name in update_info:
            self.networks.optimizer_dict[net_name].step()
        self._polyak(list(update_info))

    def _polyak(self, names=("v", "policy")):
        for name in names:
            polyak_update(self.networks.target_net_dict[name].flat_params, self.networks.net_dict[name].flat_params,
                          self.tau)

    def _value_pass(self, data) -> torch.Tensor:
        """loss_v and v's gradient; tail [loss_v | mean v | safe count 0 | safe count 1] (spil.py:182-212)."""
        nets = self.networks
        plan = self._plan(_lib.ALG_INFADP_VALUE, nets.policy, nets.v, self.forward_step, self.gamma)
        _lib.check(_lib.lib().gops_b200_plan_set_constraint(plan.handle, MODE_SPIL, 1.0))
        self._set_noise(plan, "value", data)
        return self._rollout_grad(plan, data, nets.v.flat_params, nets.policy.flat_params, nets.v.flat_params,
                                  nets.v_target.flat_params)

    def _controller(self, tail_v: torch.Tensor, data):
        """__spil_get_weight (spil.py:257-270) on the device; Kp / Ki / Kd / chance_thre are read on every call."""
        # one constraint: the second controller channel sees threshold 0 and safe count 0, so its lam stays 0
        thr = np.broadcast_to(np.asarray(self.chance_thre, dtype=np.float64), (self.n_constraint,))
        thr = np.concatenate((thr, np.zeros(2 - self.n_constraint)))
        batch = int(data["obs"].shape[0]) * self._world()[1]
        state, weights = self._ctl()
        with torch.cuda.device(state.device):
            _lib.check(_lib.lib().gops_b200_spil_controller(
                _lib.ptr(tail_v), batch, float(self.Kp), float(self.Ki), float(self.Kd), float(thr[0]), float(thr[1]),
                _lib.ptr(state), _lib.ptr(weights), _lib.stream_ptr()))

    def _policy_pass(self, data) -> torch.Tensor:
        """loss_pi and the policy's gradient; tail [loss_pi | mean R | mean Phi product 0 | 1] (spil.py:214-255)."""
        pol = self.networks.policy
        plan = self._plan(_lib.ALG_FHADP, pol, None, self.forward_step, self.gamma)
        _lib.check(_lib.lib().gops_b200_plan_set_constraint(plan.handle, MODE_SPIL, 1.0))
        _lib.check(_lib.lib().gops_b200_plan_set_spil_weights(plan.handle, _lib.ptr(self._ctl()[1])))
        self._set_noise(plan, "policy", data)
        return self._rollout_grad(plan, data, pol.flat_params, pol.flat_params, None, None)

    def _set_noise(self, plan, name: str, data):
        """pyth_mobilerobot: this pass's obstacle draws [forward_step][B][2] into the plan (kept alive until the next)."""
        if not self.noisy:
            return
        B, dev = int(data["obs"].shape[0]), self._device()
        if self.noise_override is not None:
            noise = self.noise_override[name].to(dev, torch.float32).contiguous()
            if tuple(noise.shape) != (self.forward_step, B, 2):
                raise ValueError(f"noise_override[{name!r}] must be [{self.forward_step}, {B}, 2], got {tuple(noise.shape)}")
        else:
            with torch.cuda.device(dev):
                noise = self.envmodel.unwrapped.draw_noise((self.forward_step, B, 2), dev)
        self.__dict__.setdefault("_noise_bufs", {})[name] = noise
        _lib.check(_lib.lib().gops_b200_plan_set_model_io(plan.handle, _lib.ptr(noise), None))

    def _publish(self, tail_v: torch.Tensor, tail_p: torch.Tensor, start_time: float):
        """The update's one host read (honours loss_lag): both passes' tails in one pinned buffer."""
        host = self._tail_to_host(tail_v, tail_p)
        self.tb_info[tb_tags["loss_critic"]] = host[0]
        self.tb_info[tb_tags["critic_avg_value"]] = host[1]
        self.tb_info[tb_tags["loss_actor"]] = host[GRAD_TAIL]
        self.tb_info[tb_tags["alg_time"]] = (time.time() - start_time) * 1000  # ms
