#!/usr/bin/env python
"""SPIL (chance-constrained model-based RL) on the mobile robot with one moving obstacle, trained entirely on the GPU
(counterpart of the reference's example_train/spil/spil_mlp_mobilerobot_offserial.py, with the settings of its shipped
results/SPIL/mobilerobot/config.json: [64, 64] relu DetermPolicy and StateValue, value lr 2e-3, policy lr 3e-4,
replay_batch_size 1024, forward_step 25, action limits +-[0.4, pi/3], constraint_dim 1).  Initial states are drawn
from the data env's reset law on the device (gops_b200/trainer/device_sampler.py); both passes of every update run on
the fused rollout kernel (csrc/kernel.cuh, constraint mode 4) with the obstacle noise drawn on the device, and the PI
multiplier controller runs on the device between them."""
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
    ap.add_argument("--forward_step", type=int, default=25)
    ap.add_argument("--constraint_dim", type=int, default=1)
    ap.add_argument("--replay_batch_size", type=int, default=1024)
    ap.add_argument("--max_iteration", type=int, default=80000)
    ap.add_argument("--value_learning_rate", type=float, default=2e-3)
    ap.add_argument("--policy_learning_rate", type=float, default=3e-4)
    ap.add_argument("--eval_interval", type=int, default=500)
    ap.add_argument("--log_save_interval", type=int, default=500)
    ap.add_argument("--save_folder", type=str, default=None)
    ap.add_argument("--seed", type=int, default=3736645816)
    args = vars(ap.parse_args())
    torch.manual_seed(args["seed"])
    hi = np.array([0.4, np.pi / 3], np.float32)
    kw = dict(env_id="pyth_mobilerobot", algorithm="SPIL", trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=13, action_dim=2, action_high_limit=hi, action_low_limit=-hi,
              policy_func_name="DetermPolicy", policy_func_type="MLP", policy_hidden_sizes=[64, 64],
              policy_hidden_activation="relu", policy_act_distribution="default", value_func_name="StateValue",
              value_func_type="MLP", value_hidden_sizes=[64, 64], value_hidden_activation="relu", **args)
    alg = create_alg(**kw)
    sampler = DeviceStateSampler("pyth_mobilerobot", "cuda", args["seed"])
    evaluator = DeviceEvaluator(alg, DeviceStateSampler("pyth_mobilerobot", "cuda", args["seed"] + 1),
                                num_eval_episode=256, max_step=200)
    trainer = OnDeviceSerialTrainer(alg, sampler, evaluator=evaluator, **args)
    trainer.train()
    for it, tb in trainer.history:
        print(it, {k: round(v, 4) for k, v in tb.items()})
    print("safe_prob", alg.safe_prob.tolist(), "lam", alg.lam.tolist())
