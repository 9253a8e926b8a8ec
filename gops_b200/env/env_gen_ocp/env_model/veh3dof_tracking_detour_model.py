"""env_gen_ocp 3-DoF vehicle tracking with ONE surrounding vehicle to be passed, model type (reference:
gops/env/env_gen_ocp/env_model/veh3dof_tracking_detour_model.py:13-176; the model of
example_train/fhadp/fhadp_mlp_veh3ddetour_serial.py).  On top of veh3dof_tracking: four observation entries with the
surrounding vehicle's ego-frame pose and speed (:62-76), other reward weights and termination bound (:133-163), and
info["constraint"] = 2 r - min distance of the bicircle collision model of the incoming state (:78-131) -- the constraint
provider of FHADPExterior / FHADPLagrangian / FHADPInterior.  ContextState.constraint holds the surrounding vehicle's
predictions [B, pre_horizon + 1, 1, 5] = (x, y, phi, u, delta) (context/ref_traj_with_static_obstacle.py:119-127).
Kernels: csrc/lw_detour.cuh (the fused update on the layer-wise wgmma path; `forward` = veh_step_detour_kernel)."""
import math
from typing import Union

import torch

from gops_b200.env.env_gen_ocp.env_model.veh3dof_tracking_model import Veh3DoFTrackingModel
from gops_b200.env.env_gen_ocp.pyth_base import State
from gops_b200.env.env_ocp.env_model.pyth_base_model import PythBaseModel


class Veh3DoFTrackingDetourModel(Veh3DoFTrackingModel):
    VARIANT = 1          # plan_desc.veh_detour: 1 detour, 2 surrcstr (veh3dof_tracking_surrcstr_model.py)

    def __init__(self, pre_horizon: int = 10, max_steer: float = math.pi / 6, device: Union[torch.device, str, None] = None,
                 veh_length: float = 4.8, veh_width: float = 2.0, **kwargs):
        self.pre_horizon = pre_horizon
        self.veh_length, self.veh_width = float(veh_length), float(veh_width)
        PythBaseModel.__init__(self, obs_dim=6 + 4 * pre_horizon + 4, action_dim=2, dt=0.1,
                               action_lower_bound=[-max_steer, -3], action_upper_bound=[max_steer, 3], device=device)

    def fill_plan_desc(self, desc):
        super().fill_plan_desc(desc)
        desc.veh_detour = self.VARIANT
        desc.veh_length, desc.veh_width = self.veh_length, self.veh_width

    def fill_batch(self, batch, info, f32, keep):
        super().fill_batch(batch, info, f32, keep)
        state: State = info["state"]
        surr = state.context_state.constraint
        if surr is None or surr.dim() != 4 or surr.shape[2] != 1 or surr.shape[3] < 4:
            raise KeyError("veh3dof_tracking_detour: ContextState.constraint must be the surrounding vehicle's predictions "
                           "[B, n, 1, 5] (x, y, phi, u, delta)")
        if surr.shape[3] != 5:
            surr = torch.nn.functional.pad(surr, (0, 5 - surr.shape[3]))
        surr = f32(surr)
        keep.append(surr)
        batch.surr, batch.surr_len = surr.data_ptr(), int(surr.shape[1])


    RADIUS_FACTOR = 0.5      # r = 0.5 * veh_width (veh3dof_tracking_detour_model.py:83)

    def get_constraint(self, state: State) -> torch.Tensor:
        """2 r - min distance between the two circles of the ego vehicle and of the surrounding vehicle at ContextState.t
        (reference :78-131), element-wise torch code on the caller's (device) tensors: info["constraint"] of `forward`."""
        d, r = (self.veh_length - self.veh_width) / 2, self.RADIUS_FACTOR * self.veh_width
        rs = state.robot_state
        surr = state.context_state.constraint[:, int(state.context_state.t)].to(rs.device)        # [B, n, 5]
        best = None
        for sg in (1.0, -1.0):
            ex, ey = rs[:, 0:1] + sg * d * torch.cos(rs[:, 2:3]), rs[:, 1:2] + sg * d * torch.sin(rs[:, 2:3])
            for tg in (1.0, -1.0):
                qx = surr[..., 0] + tg * d * torch.cos(surr[..., 2])
                qy = surr[..., 1] + tg * d * torch.sin(surr[..., 2])
                dist = torch.sqrt((ex - qx) ** 2 + (ey - qy) ** 2).min(dim=1, keepdim=True).values
                best = dist if best is None else torch.minimum(best, dist)
        return 2 * r - best

    def make_next_info(self, info, extra):
        next_info = super().make_next_info(info, extra)
        next_info["constraint"] = self.get_constraint(info["state"])          # of the INCOMING state (pyth_base_model.py:117-118)
        return next_info


def env_model_creator(**kwargs) -> Veh3DoFTrackingDetourModel:
    return Veh3DoFTrackingDetourModel(**kwargs)
