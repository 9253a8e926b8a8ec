"""Infinite-horizon approximate dynamic programming (INFADP), H100 edition.

Same plugin surface as the reference (gops/algorithm/infadp.py: ApproxContainer :31-64, INFADP
:67-213).  The value branch (`__compute_loss_v` :159-186) and the policy branch
(`__compute_loss_policy` :188-213) are each ONE fused CUDA kernel (no-grad / differentiated
n-step model rollout, terminal v_target, loss and flat gradient); `__update` (:121-133) is the fused
Adam step plus a fused Polyak kernel."""
__all__ = ["INFADP"]

import time
from typing import Tuple

import torch

from gops_b200 import _lib
from gops_b200.algorithm.base import AlgorithmBase, ApprBase, FusedADPMixin, target_copy
from gops_b200.create_pkg.create_apprfunc import create_apprfunc
from gops_b200.create_pkg.create_env_model import create_env_model
from gops_b200.utils.common_utils import get_apprfunc_dict
from gops_b200.utils.flat_params import FusedAdam, polyak_update
from gops_b200.utils.tensorboard_setup import tb_tags


class ApproxContainer(ApprBase):
    """v, policy and their Polyak targets + one fused Adam per trained network."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        v_args = get_apprfunc_dict("value", **kwargs)
        policy_args = get_apprfunc_dict("policy", **kwargs)
        self.v = create_apprfunc(**v_args)
        self.policy = create_apprfunc(**policy_args)
        self.v_target = target_copy(self.v)
        self.policy_target = target_copy(self.policy)
        self.policy_optimizer = FusedAdam(self.policy.flat_params, lr=kwargs["policy_learning_rate"])
        self.v_optimizer = FusedAdam(self.v.flat_params, lr=kwargs["value_learning_rate"])
        self.net_dict = {"v": self.v, "policy": self.policy}
        self.target_net_dict = {"v": self.v_target, "policy": self.policy_target}
        self.optimizer_dict = {"v": self.v_optimizer, "policy": self.policy_optimizer}
        self.scheduler_dict = {}

    def create_action_distributions(self, logits):
        return self.policy.get_act_dist(logits)


class INFADP(AlgorithmBase, FusedADPMixin):
    def __init__(self, index=0, **kwargs):
        super().__init__(index, **kwargs)
        self.networks = ApproxContainer(**kwargs)
        self.envmodel = create_env_model(**kwargs)
        self.gamma = 0.99
        self.tau = 0.005
        self.pev_step = 1
        self.pim_step = 1
        self.forward_step = 10
        self.reward_scale = kwargs.get("reward_scale", None)
        self.tb_info = dict()
        self._init_fused()

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "pev_step", "pim_step", "forward_step", "reward_scale")

    def local_update(self, data: dict, iteration: int) -> dict:
        start_time = time.time()
        # Adam + Polyak are launched behind the rollout, no sync in between
        name = "v" if iteration % (self.pev_step + self.pim_step) < self.pev_step else "policy"
        self._fuse_opt, self._opt_applied = self.networks.optimizer_dict[name], False
        try:
            update_list, tail = self.__launch_gradient(data, iteration)
        finally:
            self._fuse_opt = None
        self.__update(update_list, stepped=self._opt_applied)
        self.__publish(update_list, tail, start_time)
        return self.tb_info

    def get_remote_update_info(self, data: dict, iteration: int) -> Tuple[dict, dict]:
        start_time = time.time()
        update_list, tail = self.__launch_gradient(data, iteration)
        self.__publish(update_list, tail, start_time)
        update_info = {name: [p.grad for p in self.networks.net_dict[name].parameters()] for name in update_list}
        return self.tb_info, update_info

    def remote_update(self, update_info: dict):
        for net_name, grads in update_info.items():
            for p, grad in zip(self.networks.net_dict[net_name].parameters(), grads):
                p.grad = grad
        self.__update(list(update_info.keys()))

    def __update(self, update_list, stepped: bool = False):
        for net_name in update_list:
            if not stepped:       # on several GPUs the gradient-exchange kernel has applied the step already
                self.networks.optimizer_dict[net_name].step()
        for net_name in update_list:
            polyak_update(self.networks.target_net_dict[net_name].flat_params,
                          self.networks.net_dict[net_name].flat_params, self.tau)

    def __launch_gradient(self, data, iteration):
        """infadp.py:135-157: value branch on PEV iterations, policy branch on PIM iterations (no host sync)."""
        if iteration % (self.pev_step + self.pim_step) < self.pev_step:
            return ["v"], self.__compute_loss_v(data)
        return ["policy"], self.__compute_loss_policy(data)

    def __publish(self, update_list, tail, start_time):
        host = self._tail_to_host(tail)
        if update_list[0] == "v":
            self.tb_info[tb_tags["loss_critic"]] = host[0]
            self.tb_info[tb_tags["critic_avg_value"]] = host[1]
        else:
            self.tb_info[tb_tags["loss_actor"]] = host[0]
        self.tb_info[tb_tags["alg_time"]] = (time.time() - start_time) * 1000  # ms

    def __compute_loss_v(self, data):
        """mean((v(o) - [sum_k gamma^k r_k + (~d) gamma^n v_target(o_n)])^2), gradient -> v.grad."""
        nets = self.networks
        plan = self._plan(_lib.ALG_INFADP_VALUE, nets.policy, nets.v, self.forward_step, self.gamma)
        tail = self._rollout_grad(plan, data, nets.v.flat_params, nets.policy.flat_params, nets.v.flat_params,
                                  nets.v_target.flat_params)
        return tail

    def __compute_loss_policy(self, data):
        """-mean(sum_k gamma^k r_k + (~d) gamma^n v_target(o_n)), gradient -> policy.grad."""
        nets = self.networks
        plan = self._plan(_lib.ALG_INFADP_POLICY, nets.policy, nets.v, self.forward_step, self.gamma)
        tail = self._rollout_grad(plan, data, nets.policy.flat_params, nets.policy.flat_params, None,
                                  nets.v_target.flat_params)
        return tail
