#!/usr/bin/env python
"""RPI (relaxed policy iteration) on the oscillator with an adversarial disturbance, trained on the GPU (counterpart of
the reference's example_train/rpi/rpi_mlp_oscillatorconti_onserial.py with its settings: StateValue MLP [64, 64] elu,
Adam lr 1e-3, gamma_atte 2, 50 Newton iterations of at most 10000 policy-evaluation steps on B = 64 states).  Every
Newton iteration is one kernel launch (csrc/rpi.cu); the script logs its inner-step count and Hamiltonian norms and
saves apprfunc/apprfunc_{iteration}.pkl (the networks' state_dict, loadable by the reference's ApproxContainer)."""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gops_b200.create_pkg.create_alg import create_alg

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--max_newton_iteration", type=int, default=50)
    ap.add_argument("--max_step_update_value", type=int, default=10000)
    ap.add_argument("--learning_rate", type=float, default=1e-3)
    ap.add_argument("--gamma_atte", type=float, default=2.0)
    ap.add_argument("--value_hidden_activation", type=str, default="elu")
    ap.add_argument("--reset_batch_size", type=int, default=64)
    ap.add_argument("--apprfunc_save_interval", type=int, default=10)
    ap.add_argument("--save_folder", type=str, default=None)
    ap.add_argument("--seed", type=int, default=0)
    args = vars(ap.parse_args())
    torch.manual_seed(args["seed"])
    np.random.seed(args["seed"])
    kw = dict(env_id="pyth_oscillatorconti", algorithm="RPI", trainer="on_serial_trainer", is_adversary=True,
              value_func_name="StateValue", value_func_type="MLP", value_hidden_sizes=[64, 64],
              value_output_activation="linear", policy_func_name="DetermPolicy", policy_func_type="POLY",
              policy_act_distribution="default", sample_batch_size=args["reset_batch_size"],
              fixed_initial_state=[0.5, -0.5], initial_state_range=[1.2, 1.2], state_threshold=[5.0, 5.0],
              lower_step=100, upper_step=200, obsv_dim=2, action_dim=1, action_type="continu",
              action_high_limit=np.ones(1, np.float32), action_low_limit=-np.ones(1, np.float32), **args)
    alg = create_alg(**kw)
    save = args["save_folder"] or os.path.join("results", "RPI", time.strftime("%y%m%d-%H%M%S"))
    os.makedirs(os.path.join(save, "apprfunc"), exist_ok=True)
    t0 = time.time()
    total = 0
    for it in range(args["max_newton_iteration"]):
        info = alg.local_update(None, it)
        total += alg.num_update_value
        print(f"  n {alg.num_update_value:5d}  |H| before {alg.norm_hamiltonian_before:.6f}  after "
              f"{alg.norm_hamiltonian_after:.6f}  loss {info['Loss/Critic loss-RL iter']:.6f}  "
              f"{info['Time/Algorithm time [ms]-RL iter']:.1f} ms")
        if it % args["apprfunc_save_interval"] == 0 or it == args["max_newton_iteration"] - 1:
            sd = {k: v.detach().cpu() for k, v in alg.networks.state_dict().items()}
            torch.save(sd, os.path.join(save, "apprfunc", f"apprfunc_{it}.pkl"))
    print(f"{args['max_newton_iteration']} Newton iterations, {total} inner steps, {time.time() - t0:.2f} s")
