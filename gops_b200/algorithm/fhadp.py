"""Finite-horizon approximate dynamic programming (FHADP), H100 edition.

Same plugin surface as the reference (gops/algorithm/fhadp.py: ApproxContainer :32-55, FHADP
:58-125).  `_compute_gradient` replaces the python horizon loop + autograd of
`_compute_loss_policy` (:113-125) by ONE fused CUDA kernel (policy MLP forward, wrapper chain, env
model step, reverse sweep with hand-derived adjoints, weight-gradient reduction), followed by a
single NCCL all-reduce when run under torchrun and a fused Adam step."""
__all__ = ["FHADP"]

import time
from typing import Tuple

import torch

from gops_b200 import _lib
from gops_b200.algorithm.base import AlgorithmBase, ApprBase, FusedADPMixin
from gops_b200.create_pkg.create_apprfunc import create_apprfunc
from gops_b200.create_pkg.create_env_model import create_env_model
from gops_b200.utils.common_utils import get_apprfunc_dict
from gops_b200.utils.flat_params import FusedAdam
from gops_b200.utils.gops_typing import DataDict, InfoDict
from gops_b200.utils.tensorboard_setup import tb_tags


class ApproxContainer(ApprBase):
    """Approximate function container for FHADP: one policy network + its optimizer."""

    def __init__(self, *, policy_learning_rate: float, **kwargs):
        super().__init__(**kwargs)
        policy_args = get_apprfunc_dict("policy", **kwargs)
        self.policy = create_apprfunc(**policy_args)
        self.policy_optimizer = FusedAdam(self.policy.flat_params, lr=policy_learning_rate)
        self.optimizer_dict = {"policy": self.policy_optimizer}
        self.init_scheduler(**kwargs)

    def create_action_distributions(self, logits):
        return self.policy.get_act_dist(logits)


class FHADP(AlgorithmBase, FusedADPMixin):
    """:param int pre_horizon: env-model prediction horizon.  :param float gamma: discount factor."""

    def __init__(self, *, pre_horizon: int, gamma: float = 1.0, index: int = 0, **kwargs):
        super().__init__(index, **kwargs)
        self.networks = ApproxContainer(**kwargs)
        self.envmodel = create_env_model(**kwargs, pre_horizon=pre_horizon)
        self.pre_horizon = pre_horizon
        self.gamma = gamma
        self.tb_info = dict()
        self._init_fused()

    @property
    def adjustable_parameters(self) -> Tuple[str]:
        return ("pre_horizon", "gamma")

    def _local_update(self, data: DataDict, iteration: int) -> InfoDict:
        start_time = time.time()
        # the optimizer step is launched behind the rollout, no host sync in between
        tail = self._launch_and_step(lambda: self._launch_gradient(data), self.networks.policy_optimizer)
        self._publish(tail, start_time)
        return self.tb_info

    def get_remote_update_info(self, data: DataDict, iteration: int) -> Tuple[InfoDict, DataDict]:
        self._compute_gradient(data)
        return self.tb_info, {"grad": [p._grad for p in self.networks.policy.parameters()]}

    def _remote_update(self, update_info: DataDict):
        for p, grad in zip(self.networks.policy.parameters(), update_info["grad"]):
            p.grad = grad
        self.networks.policy_optimizer.step()

    def _compute_gradient(self, data: DataDict):
        start_time = time.time()
        self._publish(self._launch_gradient(data), start_time)

    def _publish(self, tail: torch.Tensor, start_time: float):
        self.tb_info[tb_tags["loss_actor"]] = self._tail_to_host(tail)[0]
        self.tb_info[tb_tags["alg_time"]] = (time.time() - start_time) * 1000  # ms

    def _launch_gradient(self, data: DataDict) -> torch.Tensor:
        """Loss AND gradient in one fused launch (the gradient lands in the policy's `.grad`); returns the device
        tail [loss | - | #done | -] without synchronising."""
        pol = self.networks.policy
        plan = self._plan(_lib.ALG_FHADP, pol, None, self.pre_horizon, self.gamma)
        return self._rollout_grad(plan, data, pol.flat_params, pol.flat_params, None, None)

    def _compute_loss_policy(self, data: DataDict) -> Tuple[torch.Tensor, InfoDict]:
        """Reference signature (fhadp.py:113-125): (loss, info); the gradient is already in `.grad`."""
        tail = self._launch_gradient(data)
        return tail[0], {tb_tags["loss_actor"]: tail[0].item()}
