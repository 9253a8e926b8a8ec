"""FHADP2: finite-horizon ADP with an OPEN-LOOP policy (reference gops/algorithm/fhadp2.py:20-121).

`FiniteHorizonFullPolicy` maps obs_0 to the whole action sequence; the loss is the negative discounted return of the
model rollout under that sequence (fhadp2.py:98-121).  Here: one wgmma policy evaluation (all H actions), the fused
per-step rollout kernels (forward and hand-derived adjoint, csrc/lw_rollout.cuh), one wgmma policy backward -- the
gradient lands in the policy's flat `.grad`, followed by the NCCL all-reduce (torchrun) and the fused Adam step."""
__all__ = ["FHADP2"]

import time
from typing import Tuple

import torch

from gops_b200 import _lib
from gops_b200.algorithm.base import AlgorithmBase, ApprBase, FusedADPMixin
from gops_b200.create_pkg.create_apprfunc import create_apprfunc
from gops_b200.create_pkg.create_env_model import create_env_model
from gops_b200.utils.common_utils import get_apprfunc_dict
from gops_b200.utils.flat_params import FusedAdam
from gops_b200.utils.tensorboard_setup import tb_tags


class ApproxContainer(ApprBase):
    """One open-loop policy network + its optimizer (fhadp2.py:31-47)."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        policy_args = get_apprfunc_dict("policy", **kwargs)
        self.policy = create_apprfunc(**policy_args)
        self.policy_optimizer = FusedAdam(self.policy.flat_params, lr=kwargs["policy_learning_rate"])
        self.optimizer_dict = {"policy": self.policy_optimizer}
        self.init_scheduler(**kwargs)

    def create_action_distributions(self, logits):
        return self.policy.get_act_dist(logits)


class FHADP2(AlgorithmBase, FusedADPMixin):
    def __init__(self, index=0, **kwargs):
        super().__init__(index, **kwargs)
        self.networks = ApproxContainer(**kwargs)
        self.envmodel = create_env_model(**kwargs)
        self.forward_step = kwargs["pre_horizon"]
        self.gamma = 1.0
        self.tb_info = dict()
        self._init_fused()

    @property
    def adjustable_parameters(self):
        return ("forward_step", "gamma")

    def _local_update(self, data, iteration: int):
        start_time = time.time()
        tail = self._launch_and_step(lambda: self._launch_gradient(data), self.networks.policy_optimizer)
        self._publish(tail, start_time)
        return self.tb_info

    def get_remote_update_info(self, data: dict, iteration: int) -> Tuple[dict, dict]:
        start_time = time.time()
        self._publish(self._launch_gradient(data), start_time)
        return self.tb_info, {"grad": [p._grad for p in self.networks.policy.parameters()]}

    def _remote_update(self, update_info: dict):
        for p, grad in zip(self.networks.policy.parameters(), update_info["grad"]):
            p.grad = grad
        self.networks.policy_optimizer.step()

    def _publish(self, tail: torch.Tensor, start_time: float):
        self.tb_info[tb_tags["loss_actor"]] = self._tail_to_host(tail)[0]
        self.tb_info[tb_tags["alg_time"]] = (time.time() - start_time) * 1000  # ms

    def _launch_gradient(self, data) -> torch.Tensor:
        pol = self.networks.policy
        if self.forward_step != pol.pre_horizon:
            raise RuntimeError("FHADP2: forward_step must equal the policy's pre_horizon (one action block per step)")
        plan = self._plan(_lib.ALG_FHADP, pol, None, self.forward_step, self.gamma, open_loop=True)
        return self._rollout_grad(plan, data, pol.flat_params, pol.flat_params, None, None)
