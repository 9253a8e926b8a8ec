"""CPU oracle of pyth_mobilerobot (gops/env/env_ocp/env_model/pyth_mobilerobot_model.py) -- TEST INFRASTRUCTURE, not the
product.

A restatement in PyTorch (fp32 or fp64) of PythMobilerobotModel.forward (:61-122, Robot.f_xu :136-178, tracking_error
:180-195) that takes the obstacle noise as an input instead of drawing it from NumPy's global RNG, for the wrapper chain
and the SPIL passes of oracle/gops_oracle.py and oracle/spil_oracle.py.  `replay_normal` feeds given draws to the
unmodified reference in place of np.random.normal."""
import contextlib
from typing import List

import numpy as np
import torch

from oracle import gops_oracle as orc

STD = (0.03, 0.02)          # the obstacle's std_type["obs"]; the ego's draws have std 0


class MobileRobotModel(orc.BaseModel):
    """`noise`: a list of [B, 2] tensors, one per call of `step` (float32 draws normal(0, STD), applied times 0.5)."""
    obs_dim, action_dim, dt = 13, 2, 0.2

    def __init__(self, dtype=torch.float32, noise: List[torch.Tensor] = None, **_):
        self.dtype = dtype
        lo = [-30, -30, -2 * np.pi, -1, -np.pi / 2] + [-30, -np.pi, -2] + [-30, -30, -2 * np.pi, -1, -np.pi / 2]
        hi = [60, 30, 2 * np.pi, 1, np.pi / 2] + [30, np.pi, 2] + [30, 30, 2 * np.pi, 1, np.pi / 2]
        # the reference's bounds are float32 tensors whatever the oracle's dtype
        f32 = lambda v: torch.tensor(v, dtype=torch.float32).to(dtype).tolist()
        self._bounds(f32(lo), f32(hi), f32([-0.4, -np.pi / 3]), f32([0.4, np.pi / 3]), dtype=dtype)
        self.noise = list(noise) if noise is not None else []
        self.calls = 0

    @staticmethod
    def f_xu(s, cmd, noise, T=0.2):
        v, w = s[:, 3], s[:, 4]
        dv = torch.clamp(cmd[:, 0] - v, -1.8 * T, 1.8 * T)
        dw = torch.clamp(cmd[:, 1] - w, -0.8 * T, 0.8 * T)
        vc = torch.clamp(v + dv, -0.4, 0.4) + noise[:, 0] * 0.5
        wc = torch.clamp(w + dw, -np.pi / 2, np.pi / 2) + noise[:, 1] * 0.5
        return torch.stack([s[:, 0] + T * torch.cos(s[:, 2]) * vc, s[:, 1] + T * torch.sin(s[:, 2]) * vc,
                            s[:, 2] + T * wc, vc, wc], 1)

    def step(self, obs, action, done, info):
        n = self.noise[self.calls].to(obs.dtype)
        self.calls += 1
        zero = torch.zeros_like(n)
        ego = self.f_xu(obs[:, :5], action, zero)
        err = torch.stack([ego[:, 1], ego[:, 2], ego[:, 3] - 0.3], 1)      # path y = 0, phi = 0
        other = self.f_xu(obs[:, 8:13], obs[:, 11:13], n)
        nxt = torch.cat([ego, err, other], 1)
        c = (0.74 / 2 + 0.74 / 2 + 0.15) - torch.sqrt(torch.square(other[:, 0] - ego[:, 0]) +
                                                      torch.square(other[:, 1] - ego[:, 1]))
        r = (-1.4 * torch.square(err[:, 0]) - 1 * torch.square(err[:, 1]) - 16 * torch.square(err[:, 2])
             - 0.2 * torch.square(action[:, 0]) - 0.5 * torch.square(action[:, 1]))
        d = (ego[:, 0] < -2) | (torch.abs(ego[:, 1]) > 4) | (c > 0.15)
        return nxt, r, d, {"constraint": c.unsqueeze(1)}


def create_env_model(noise, dtype=torch.float32, **wrap) -> orc.WrappedModel:
    """The default wrapper chain of create_env_model around the oracle model (ScaleAction, ClipAction, ClipObservation,
    MaskAtDone), with `noise` consumed one [B, 2] entry per forward."""
    return orc.WrappedModel(MobileRobotModel(dtype=dtype, noise=noise), **wrap)


def draw(shape, seed: int) -> np.ndarray:
    """float32(normal(0, STD)) draws [..., 2] from NumPy's legacy RNG, as the reference forms them."""
    rs = np.random.RandomState(seed)
    return np.stack([rs.normal(0, STD[0], shape), rs.normal(0, STD[1], shape)], -1).astype(np.float32)


@contextlib.contextmanager
def replay_normal(noise_steps):
    """Within the block, the reference's np.random.normal returns the given draws: per model step four calls in f_xu's
    order (ego v, ego w with std 0 -> zeros; obstacle v, w -> noise_steps[k][:, 0], [:, 1])."""
    real = np.random.normal
    seq = []
    for n in noise_steps:
        n = np.asarray(n, dtype=np.float32)
        seq += [None, None, n[:, 0].astype(np.float64), n[:, 1].astype(np.float64)]
    it = iter(seq)

    def fake(loc=0.0, scale=1.0, size=None):
        v = next(it)
        if v is None:
            assert scale == 0, scale
            return np.zeros(size)
        assert np.asarray(size).tolist() == [len(v)] or size == len(v), (size, len(v))
        return v.copy()

    np.random.normal = fake
    try:
        yield
    finally:
        np.random.normal = real
