"""Oscillator with an adversarial disturbance, model type (reference:
gops/env/env_ocp/env_model/pyth_oscillatorconti_model.py): the continuous-time zero-sum (H-infinity) task of RPI.

    dx0 = -0.25 x0
    dx1 = 0.5 x0^2 x1 - x1^3 / (2 gamma_atte^2) - 0.5 x1 + x0 u + x1 w
    c   = x0^2 + x1^2 + u^2 - gamma_atte^2 w^2

The action is [u, w] with bounds [-5, 5] and [-1/gamma_atte, 1/gamma_atte].  RPI's hot path (sampling, the Hamiltonian
loss and its stopping test) runs in gops_b200/csrc/rpi.cu, which evaluates this model on the device; the methods here
are the model's host-side surface (`forward` for evaluation and tests, `reset` / `step` as the reference's sampler,
the control-affine parts f_x / g_x / k_x and the closed-form best_act / worst_adv)."""
from typing import Tuple, Union

import numpy as np
import torch

from gops_b200.env.env_ocp.env_model.pyth_base_model import PythBaseModel
from gops_b200.utils.gops_typing import InfoDict


class PythOscillatorcontiModel(PythBaseModel):
    def __init__(self, device: Union[torch.device, str, None] = None, **kwargs):
        self.is_adversary = kwargs["is_adversary"]
        self.sample_batch_size = kwargs["reset_batch_size"]
        self.state_dim = 2
        self.adversary_dim = 1
        self.gamma = 1
        self.gamma_atte = kwargs["gamma_atte"]
        self.fixed_initial_state = kwargs["fixed_initial_state"]
        self.initial_state_range = list(kwargs["initial_state_range"])
        self.state_threshold = list(kwargs["state_threshold"])
        self.min_action, self.max_action = [-5.0], [5.0]
        self.min_adv_action, self.max_adv_action = [-1.0 / self.gamma_atte], [1.0 / self.gamma_atte]
        lb_action = self.min_action + (self.min_adv_action if self.is_adversary else [])
        hb_action = self.max_action + (self.max_adv_action if self.is_adversary else [])
        th = self.state_threshold
        # action_dim is the control's dimension (1); the adversary enlarges the action bounds only, as in the reference
        super().__init__(obs_dim=2, action_dim=1, dt=1 / 200, obs_lower_bound=[-th[0], -th[1]],
                         obs_upper_bound=[th[0], th[1]], action_lower_bound=lb_action, action_upper_bound=hb_action,
                         device="cpu")
        self.Q = torch.eye(self.state_dim)
        self.R = torch.eye(self.action_dim)
        self.ones_ = torch.ones(self.sample_batch_size)
        self.zeros_ = torch.zeros(self.sample_batch_size)
        self.parallel_state = None
        self.lower_step = kwargs["lower_step"]
        self.upper_step = kwargs["upper_step"]
        self.max_step_per_episode = self.max_step()
        self.step_per_episode = self.initial_step()

    def max_step(self) -> torch.Tensor:
        """floor(U[lower_step, upper_step)) per sample, drawn from NumPy's global RNG."""
        return torch.from_numpy(np.floor(np.random.uniform(self.lower_step, self.upper_step, [self.sample_batch_size])))

    def initial_step(self) -> torch.Tensor:
        return torch.zeros(self.sample_batch_size)

    def reset(self) -> torch.Tensor:
        """U[-r_i, r_i] per component: all first components, then all second components (NumPy's global RNG)."""
        r0, r1 = self.initial_state_range
        a = np.random.uniform(-r0, r0, [self.sample_batch_size, 1])
        b = np.random.uniform(-r1, r1, [self.sample_batch_size, 1])
        return torch.from_numpy(np.concatenate([a, b], axis=1)).float()

    def _dynamics(self, state, u, w):
        x0, x1 = state[:, 0], state[:, 1]
        d0 = -0.25 * x0
        d1 = (0.5 * torch.mul(x0 ** 2, x1) - 1 / (2 * self.gamma_atte ** 2) * x1 ** 3 - 0.5 * x1
              + torch.mul(x0, u) + torch.mul(x1, w))
        cost = self.Q[0][0] * x0 ** 2 + self.Q[1][1] * x1 ** 2 + self.R[0][0] * u ** 2 - self.gamma_atte ** 2 * w ** 2
        return torch.stack([d0, d1], dim=-1), cost

    def step(self, action: torch.Tensor):
        """The reference's sampler step on `parallel_state` with the RAW action (no wrapper)."""
        delta, cost = self._dynamics(self.parallel_state, action[:, 0], action[:, 1])
        self.parallel_state = self.parallel_state + delta * self.dt
        th = self.state_threshold
        done = (abs(self.parallel_state[:, 0]) > th[0]) | (abs(self.parallel_state[:, 1]) > th[1])
        self.step_per_episode += 1
        info = {"TimeLimit.truncated": self.step_per_episode > self.max_step_per_episode}
        return self.parallel_state, cost, done, info

    def forward(self, obs: torch.Tensor, action: torch.Tensor, done: torch.Tensor, info: InfoDict
                ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, InfoDict]:
        u = action[:, 0]
        w = action[:, 1] if self.is_adversary else torch.zeros_like(u)
        delta, cost = self._dynamics(obs, u, w)
        return obs + delta * self.dt, -cost, obs.new_zeros(obs.shape[0], dtype=torch.bool), {"delta_state": delta}

    def f_x(self, state, batch_size):
        fx = torch.zeros((batch_size, self.state_dim))
        fx[:, 0] = -0.25 * state[:, 0]
        fx[:, 1] = (0.5 * torch.mul(state[:, 0] ** 2, state[:, 1]) - 1 / (2 * self.gamma_atte ** 2) * state[:, 1] ** 3
                    - 0.5 * state[:, 1])
        return fx if batch_size > 1 else fx.t()

    def g_x(self, state, batch_size):
        gx = torch.zeros((batch_size, self.state_dim, self.action_dim))
        gx[:, 1, 0] = state[:, 0]
        return gx if batch_size > 1 else gx[0]

    def k_x(self, state, batch_size):
        kx = torch.zeros((batch_size, self.state_dim, self.adversary_dim))
        kx[:, 1, 0] = state[:, 1]
        return kx if batch_size > 1 else kx[0]

    def best_act(self, state, delta_value):
        """u* = -0.5 R^-1 g(x)^T dV/dx."""
        gx = self.g_x(state, state.shape[0]).reshape(state.shape[0], self.state_dim, self.action_dim)
        act = -0.5 * torch.matmul(self.R.inverse(), torch.bmm(gx.transpose(1, 2), delta_value[:, :, None])).squeeze(-1)
        return act.detach()

    def worst_adv(self, state, delta_value):
        """w* = 0.5 / gamma_atte^2 k(x)^T dV/dx."""
        kx = self.k_x(state, state.shape[0]).reshape(state.shape[0], self.state_dim, self.adversary_dim)
        return (0.5 / (self.gamma_atte ** 2) * torch.bmm(kx.transpose(1, 2), delta_value[:, :, None]).squeeze(-1)).detach()


def env_model_creator(**kwargs):
    """make env model `pyth_oscillatorconti`"""
    return PythOscillatorcontiModel(**kwargs)
