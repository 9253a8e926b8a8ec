"""Mobile robot with one moving obstacle, model type (reference: gops/env/env_ocp/env_model/pyth_mobilerobot_model.py).
The dynamics (Robot.f_xu :136-178, tracking_error :180-195), reward, done and the obstacle-distance constraint, with their
adjoint, are implemented in gops_b200/csrc/models_robot.cuh (ModelMobileRobot).

The reference draws the obstacle's command noise from NumPy's global RNG inside `forward`.  Here the draws are an input
of the kernels: `draw_noise` fills a device buffer with float32(normal(0, (0.03, 0.02))) from a generator this
descriptor owns (one draw per call), unless `noise_override` holds given draws ([B, 2] for `forward`).  The rollout
passes and `forward` draw from two generators, so evaluating a policy through `forward` leaves the training noise
stream as it is."""
from typing import Optional, Tuple, Union

import numpy as np
import torch

from gops_b200 import _lib
from gops_b200.env.env_ocp.env_model.pyth_base_model import PythBaseModel

OBSTACLE_NOISE_STD = (0.03, 0.02)      # Robot.f_xu std_type["obs"]: the obstacle's v, w


class PythMobilerobotModel(PythBaseModel):
    MODEL_KIND = _lib.MODEL_MOBILEROBOT

    def __init__(self, device: Union[torch.device, str, None] = None, **kwargs):
        self.n_obstacle = 1
        self.safe_margin = 0.15
        self.constraint_dim = self.n_obstacle
        lb_state = [-30, -30, -2 * np.pi, -1, -np.pi / 2] + [-30, -np.pi, -2] + [-30, -30, -2 * np.pi, -1, -np.pi / 2]
        hb_state = [60, 30, 2 * np.pi, 1, np.pi / 2] + [30, np.pi, 2] + [30, 30, 2 * np.pi, 1, np.pi / 2]
        super().__init__(obs_dim=13, action_dim=2, dt=0.2, obs_lower_bound=lb_state, obs_upper_bound=hb_state,
                         action_lower_bound=[-0.4, -np.pi / 3], action_upper_bound=[0.4, np.pi / 3], device=device)
        self.noise_override: Optional[torch.Tensor] = None

    def draw_noise(self, shape: Tuple[int, ...], dev, stream: str = "rollout") -> torch.Tensor:
        """float32 [..., 2] obstacle draws on `dev`: n ~ normal(0, std) per entry (the kernels apply the 0.5).
        stream: "rollout" (the SPIL passes) or "forward" (envmodel.forward), each with a generator of its own."""
        dev = torch.device(dev)
        gens = self.__dict__.setdefault("_gens", {})
        gen = gens.get((stream, dev))
        if gen is None:
            seed = int(torch.initial_seed() % (2 ** 31)) + (1 if stream == "forward" else 0)
            gen = gens[(stream, dev)] = torch.Generator(device=dev).manual_seed(seed)
        n = torch.randn(shape, generator=gen, device=dev, dtype=torch.float32)
        return n.mul_(torch.tensor(OBSTACLE_NOISE_STD, dtype=torch.float32, device=dev))

    def model_io(self, B: int, dev):
        """(noise [B, 2], constraint out [B, 1]) of one `forward`."""
        if self.noise_override is not None:
            noise = self.noise_override.to(dev, torch.float32).contiguous()
            if tuple(noise.shape) != (B, 2):
                raise ValueError(f"noise_override must be [{B}, 2], got {tuple(noise.shape)}")
        else:
            noise = self.draw_noise((B, 2), dev, "forward")
        return noise, torch.empty((B, 1), dtype=torch.float32, device=dev)

    def make_next_info(self, info, extra):
        return {"constraint": extra["constraint"]}


def env_model_creator(**kwargs):
    """make env model `pyth_mobilerobot`"""
    return PythMobilerobotModel(kwargs.get("device", None))
