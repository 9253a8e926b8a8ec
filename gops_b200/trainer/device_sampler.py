"""Batched initial-state samplers that live on the GPU (SURVEY.md 8(f) N2, the caller side of the fused update).

The reference fills its replay buffer by resetting ONE NumPy data env at a time on the CPU
(gops/trainer/sampler/base.py:101-187 -> env.reset) and copies a batch to the GPU for every update.  The model-based
ADP algorithms only consume the batch's INITIAL STATES (`obs`, `done` and the vehicle `info` entries), so the same
reset distributions are drawn here for a whole batch at once, directly in device memory:

  pyth_idpendulum     uniform box                        pyth_idpendulum.py:36-38, pyth_base_env.py:61-65
  pyth_lq             N(init_mean, init_std)             lq_base.py:151-155, lq_configs.py
  pyth_veh3dofconti   ref_time ~ 20 U, path ~ U{0..3}, speed ~ U{0,1}, tracking error ~ U(+-[2,1,pi/6,2,.1,.1]),
                      P+1 reference points               pyth_veh3dofconti.py:144-191
  veh3dof_tracking    same law, 2P+1 reference points, t = 0        env_gen_ocp/context/ref_traj.py:25-53,
                                                                    env_gen_ocp/veh3dof_tracking.py:58-101

Plumbing only (torch RNG + elementwise torch ops on the device); the reference-trajectory formulas are those of
gops/env/env_ocp/resources/ref_traj_model.py:54-232 with the default parameters of ref_traj_data.py:19-37.
"""
import math
from typing import Dict

import numpy as np
import torch

TWO_PI = 2.0 * math.pi


def _gen(device, seed):
    return torch.Generator(device=device).manual_seed(int(seed))


class RefTrajectory:
    """Analytic multi-path reference: path 0 sine, 1 double lane change, 2 triangle, 3 circle; speed 0 sine, 1 constant."""

    def __init__(self, sine_A=1.5, sine_omega=TWO_PI / 10, sine_phi=0.0, dl_t=(5.0, 9.0, 14.0, 18.0), dl_y=(0.0, 3.5),
                 tri_A=3.0, tri_T=10.0, circ_r=100.0, sp_A=1.0, sp_omega=TWO_PI / 10, sp_phi=0.0, sp_b=5.0, sp_const=5.0):
        self.__dict__.update(locals())

    def speed(self, t, spd):
        return torch.where(spd == 0, self.sp_A * torch.sin(self.sp_omega * t + self.sp_phi) + self.sp_b,
                           torch.full_like(t, self.sp_const))

    def arc(self, t, spd):
        """integral of the speed profile from 0 to t"""
        k = self.sp_A / self.sp_omega
        return torch.where(spd == 0, -k * torch.cos(self.sp_omega * t + self.sp_phi) + self.sp_b * t + k * math.cos(self.sp_phi),
                           self.sp_const * t)

    def xy(self, t, path, spd):
        s = self.arc(t, spd)
        x = torch.where(path == 3, self.circ_r * torch.sin(s / self.circ_r), s)
        t1, t2, t3, t4 = self.dl_t
        y1, y2 = self.dl_y
        up, down = (y2 - y1) / (t2 - t1) * (t - t1) + y1, (y1 - y2) / (t4 - t3) * (t - t3) + y2
        lane = torch.where(t <= t1, torch.full_like(t, y1), torch.where(t <= t2, up, torch.where(
            t <= t3, torch.full_like(t, y2), torch.where(t <= t4, down, torch.full_like(t, y1)))))
        r = torch.remainder(t, self.tri_T)
        k = 2 * self.tri_A / self.tri_T
        tri = torch.where(r <= self.tri_T / 2, k * r, -k * (r - self.tri_T))
        y = torch.where(path == 0, self.sine_A * torch.sin(self.sine_omega * t + self.sine_phi),
                        torch.where(path == 1, lane, torch.where(path == 2, tri,
                                                                 self.circ_r * (torch.cos(s / self.circ_r) - 1))))
        return x, y

    def point(self, t, path, spd):
        """[..., 4] = (x, y, phi, u) at time t; phi by the reference's forward difference with dt = 1e-3."""
        x0, y0 = self.xy(t, path, spd)
        x1, y1 = self.xy(t + 1e-3, path, spd)
        return torch.stack((x0, y0, torch.atan2(y1 - y0, x1 - x0), self.speed(t, spd)), -1)


def wrap_angle(a):
    return torch.remainder(a + math.pi, TWO_PI) - math.pi


def ego_observation(state, ref_points):
    """obs = [dx0, dy0, dphi0, du0, v, w, (dx, dy, dphi, du)_{1..P}] in the ego frame (pyth_veh3dofconti_model.py:147-203)."""
    x, y, phi = state[:, 0:1], state[:, 1:2], state[:, 2:3]
    c, s = torch.cos(phi), torch.sin(phi)
    rx, ry = ref_points[..., 0] - x, ref_points[..., 1] - y
    ex, ey = rx * c + ry * s, -rx * s + ry * c
    ephi = wrap_angle(ref_points[..., 2] - phi)
    eu = ref_points[..., 3] - state[:, 3:4]
    e = torch.stack((ex, ey, ephi, eu), -1)                  # [B, P+1, 4]
    return torch.cat((e[:, 0], state[:, 4:6], e[:, 1:].reshape(e.shape[0], -1)), 1)


def sample_idpendulum(batch, device, seed=0, gen=None) -> Dict[str, torch.Tensor]:
    g = gen or _gen(device, seed)
    high = torch.tensor([5, 0.1, 0.1, 0.3, 0.3, 0.3], dtype=torch.float32, device=device)
    return {"obs": (torch.rand(batch, 6, generator=g, device=device) * 2 - 1) * high,
            "done": torch.zeros(batch, device=device)}


def sample_mobilerobot(batch, device, seed=0, gen=None) -> Dict[str, torch.Tensor]:
    """The data env's uniform reset box (env_ocp/pyth_mobilerobot.py:31-53) with the tracking error of the drawn robot
    state against the path y = 0 (its `reset`): [y, theta, v - 0.3]."""
    g = gen or _gen(device, seed)
    f32 = lambda v: torch.tensor(np.asarray(v, dtype=np.float32), device=device)
    low = f32([0, -1, -0.6, 0, 0] + [0, 0, 0] + [3.5, -3, np.pi / 2 - 0.3, 0.0, 0])
    high = f32([2.7, 1, 0.6, 0.3, 0] + [0, 0, 0] + [6, 3, np.pi / 2 + 0.3, 0.5, 0])
    obs = low + torch.rand(batch, 13, generator=g, device=device) * (high - low)
    obs[:, 5], obs[:, 6], obs[:, 7] = obs[:, 1], obs[:, 2], obs[:, 3] - np.float32(0.3)
    return {"obs": obs, "done": torch.zeros(batch, device=device)}


def sample_lq(batch, lq_config, device, seed=0, gen=None) -> Dict[str, torch.Tensor]:
    from gops_b200.env.env_ocp.resources import lq_configs
    cfg = getattr(lq_configs, "config_" + lq_config) if isinstance(lq_config, str) else lq_config
    g = gen or _gen(device, seed)
    mean = torch.tensor(cfg["init_mean"], dtype=torch.float32, device=device)
    std = torch.tensor(cfg["init_std"], dtype=torch.float32, device=device)
    return {"obs": mean + std * torch.randn(batch, mean.numel(), generator=g, device=device),
            "done": torch.zeros(batch, device=device)}


def _vehicle_draw(batch, n_points, device, g, traj):
    t0 = 20.0 * torch.rand(batch, generator=g, device=device)
    path = torch.randint(0, 4, (batch,), generator=g, device=device).float()
    spd = torch.randint(0, 2, (batch,), generator=g, device=device).float()
    tt = t0[:, None] + 0.1 * torch.arange(n_points, device=device, dtype=torch.float32)[None, :]
    ref = traj.point(tt, path[:, None].expand_as(tt), spd[:, None].expand_as(tt))            # [B, n, 4]
    high = torch.tensor([2, 1, math.pi / 6, 2, 0.1, 0.1], dtype=torch.float32, device=device)
    delta = (torch.rand(batch, 6, generator=g, device=device) * 2 - 1) * high
    state = torch.cat((ref[:, 0] + delta[:, :4], delta[:, 4:]), 1)
    state[:, 2] = wrap_angle(state[:, 2])
    return t0, path, spd, ref, state


def sample_veh3dofconti(batch, pre_horizon, device, seed=0, gen=None, traj=None) -> Dict[str, torch.Tensor]:
    g = gen or _gen(device, seed)
    t0, path, spd, ref, state = _vehicle_draw(batch, pre_horizon + 1, device, g, traj or RefTrajectory())
    return {"obs": ego_observation(state, ref), "done": torch.zeros(batch, device=device), "state": state,
            "ref_points": ref.contiguous(), "path_num": path, "u_num": spd, "ref_time": t0}


def sample_veh3dof_tracking(batch, pre_horizon, device, seed=0, gen=None, traj=None) -> Dict[str, torch.Tensor]:
    from gops_b200.env.env_gen_ocp.pyth_base import ContextState, State
    g = gen or _gen(device, seed)
    _, _, _, ref, state = _vehicle_draw(batch, 2 * pre_horizon + 1, device, g, traj or RefTrajectory())
    return {"obs": ego_observation(state, ref[:, :pre_horizon + 1]), "done": torch.zeros(batch, device=device),
            "state": State(robot_state=state, context_state=ContextState(reference=ref.contiguous(), t=0))}


def sample_veh3dof_tracking_detour(batch, pre_horizon, device, seed=0, gen=None, traj=None) -> Dict[str, torch.Tensor]:
    """veh3dof_tracking plus the surrounding vehicle of the detour task: a STATIC vehicle 20 m ahead of the reference's
    first point and 1 m to its left (env_gen_ocp/context/ref_traj_with_static_obstacle.py:76-97), predicted over
    pre_horizon + 1 points as [x, y, phi, u, delta] (:119-127) in ContextState.constraint [B, P + 1, 1, 5]; the
    observation gets its ego-frame pose and speed appended (env_model/veh3dof_tracking_detour_model.py:62-76)."""
    from gops_b200.env.env_gen_ocp.pyth_base import ContextState, State
    g = gen or _gen(device, seed)
    _, _, _, ref, state = _vehicle_draw(batch, 2 * pre_horizon + 1, device, g, traj or RefTrajectory())
    surr0 = torch.stack((ref[:, 0, 0] + 20.0, ref[:, 0, 1] + 1.0, torch.zeros(batch, device=device),
                         torch.zeros(batch, device=device), torch.zeros(batch, device=device)), 1)
    surr = surr0[:, None, None, :].expand(batch, pre_horizon + 1, 1, 5).contiguous()
    sx, sy = surr0[:, 0:1] - state[:, 0:1], surr0[:, 1:2] - state[:, 1:2]
    c, s = torch.cos(state[:, 2:3]), torch.sin(state[:, 2:3])
    surr_obs = torch.cat((sx * c + sy * s, -sx * s + sy * c, wrap_angle(surr0[:, 2:3] - state[:, 2:3]), surr0[:, 3:4]), 1)
    obs = torch.cat((ego_observation(state, ref[:, :pre_horizon + 1]), surr_obs), 1)
    return {"obs": obs, "done": torch.zeros(batch, device=device),
            "state": State(robot_state=state, context_state=ContextState(reference=ref.contiguous(), constraint=surr, t=0))}
