#!/usr/bin/env python
"""SPIL (chance-constrained model-based RL) on the error-constrained vehicle tracking task, trained entirely on the GPU
(counterpart of the reference's example_train/spil/spil_mlp_veh3dofconti_errcstr_offserial.py: pyth_veh3dofconti_errcstr,
pre_horizon 10, forward_step 10, [64, 64] relu DetermPolicy and StateValue, lr 1e-3 for both, y_error_tol 0.1,
constraint_dim 2).  Initial states are drawn on the device (gops_b200/trainer/device_sampler.py); both passes of every
update run on the fused rollout kernel (csrc/kernel.cuh, constraint mode 4) and the PI multiplier controller runs on the
device between them."""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gops_b200.create_pkg.create_alg import create_alg
from gops_b200.trainer.device_trainer import DeviceEvaluator, DeviceStateSampler, OnDeviceSerialTrainer

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--pre_horizon", type=int, default=10)
    ap.add_argument("--forward_step", type=int, default=10)
    ap.add_argument("--y_error_tol", type=float, default=0.1)
    ap.add_argument("--constraint_dim", type=int, default=2)
    ap.add_argument("--reward_scale", type=float, default=1.0)
    ap.add_argument("--replay_batch_size", type=int, default=4096)
    ap.add_argument("--max_iteration", type=int, default=4000)
    ap.add_argument("--value_learning_rate", type=float, default=1e-3)
    ap.add_argument("--policy_learning_rate", type=float, default=1e-3)
    ap.add_argument("--eval_interval", type=int, default=100)
    ap.add_argument("--log_save_interval", type=int, default=100)
    ap.add_argument("--save_folder", type=str, default=None)
    ap.add_argument("--seed", type=int, default=12345)
    args = vars(ap.parse_args())
    torch.manual_seed(args["seed"])
    P = args["pre_horizon"]
    kw = dict(env_id="pyth_veh3dofconti_errcstr", algorithm="SPIL", trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=6 + 4 * P, action_dim=2, action_high_limit=np.ones(2, np.float32),
              action_low_limit=-np.ones(2, np.float32), policy_func_name="DetermPolicy", policy_func_type="MLP",
              policy_hidden_sizes=[64, 64], policy_hidden_activation="relu", policy_act_distribution="default",
              value_func_name="StateValue", value_func_type="MLP", value_hidden_sizes=[64, 64],
              value_hidden_activation="relu", **args)
    alg = create_alg(**kw)
    sampler = DeviceStateSampler("pyth_veh3dofconti_errcstr", "cuda", args["seed"], pre_horizon=P)
    evaluator = DeviceEvaluator(alg, DeviceStateSampler("pyth_veh3dofconti_errcstr", "cuda", args["seed"] + 1, pre_horizon=P),
                                num_eval_episode=256, max_step=200)
    trainer = OnDeviceSerialTrainer(alg, sampler, evaluator=evaluator, **args)
    trainer.train()
    for it, tb in trainer.history:
        print(it, {k: round(v, 4) for k, v in tb.items()})
    print("safe_prob", alg.safe_prob.tolist(), "lam", alg.lam.tolist())
