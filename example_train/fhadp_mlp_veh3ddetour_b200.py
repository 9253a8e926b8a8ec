#!/usr/bin/env python
"""Interior-point FHADP on the vehicle detour task, trained entirely on the GPU (counterpart of the reference's
example_train/fhadp/fhadp_mlp_veh3ddetour_serial.py: FHADPInterior, veh3dof_tracking_detour, pre_horizon 30,
[256, 256] elu policy, lr 1e-3).  States, references and the surrounding vehicle's predictions are drawn on the device
(gops_b200/trainer/device_sampler.py); the update runs on the layer-wise wgmma path (csrc/lw_detour.cuh)."""
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
    ap.add_argument("--algorithm", type=str, default="FHADPInterior",
                    choices=["FHADP", "FHADPInterior", "FHADPExterior", "FHADPLagrangian"])
    ap.add_argument("--pre_horizon", type=int, default=30)
    ap.add_argument("--replay_batch_size", type=int, default=4096)
    ap.add_argument("--max_iteration", type=int, default=2000)
    ap.add_argument("--policy_learning_rate", type=float, default=1e-3)
    ap.add_argument("--eval_interval", type=int, default=100)
    ap.add_argument("--save_folder", type=str, default=None)
    ap.add_argument("--seed", type=int, default=12345)
    args = vars(ap.parse_args())
    torch.manual_seed(args["seed"])
    P = args["pre_horizon"]
    kw = dict(env_id="veh3dof_tracking_detour", trainer="off_serial_trainer", use_gpu=True, action_type="continu",
              obsv_dim=6 + 4 * P + 4, action_dim=2, action_high_limit=np.ones(2, np.float32),
              action_low_limit=-np.ones(2, np.float32), policy_func_name="FiniteHorizonPolicy", policy_func_type="MLP",
              policy_hidden_sizes=[256, 256], policy_hidden_activation="elu", policy_act_distribution="default",
              value_func_type="MLP", **args)
    alg = create_alg(**kw)
    sampler = DeviceStateSampler("veh3dof_tracking_detour", "cuda", args["seed"], pre_horizon=P)
    # the model-type context carries P + 1 predictions of the surrounding vehicle: an evaluation episode is P - 1 steps
    evaluator = DeviceEvaluator(alg, DeviceStateSampler("veh3dof_tracking_detour", "cuda", args["seed"] + 1, pre_horizon=P),
                                num_eval_episode=256, max_step=P - 1)
    trainer = OnDeviceSerialTrainer(alg, sampler, log_save_interval=100, evaluator=evaluator, **args)
    trainer.train()
    for it, tb in trainer.history:
        print(it, {k: round(v, 4) for k, v in tb.items()})
