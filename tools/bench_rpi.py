"""Time RPI's Newton iterations on pyth_oscillatorconti with the reference example's settings (StateValue [64, 64] elu,
B = 64, lr 1e-3, gamma_atte 2, seed 0): the GPU path (one gops_b200_rpi_newton launch per iteration) and the
unmodified reference's RPI.local_update on the host CPU (from oracle/_ref, built by __graft_entry__.build()), each for
the same number of Newton iterations.  GPU: a host clock around each iteration, which ends in its one device read;
the GPU run also repeats at B = 512 (a cluster of 8 CTAs).  Reports inner steps/s and ms per Newton iteration, the card
name and power limit, and writes the JSON to --out.

    python tools/bench_rpi.py --iters 13 --out results/bench_rpi.json"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_leg(iters, B):
    from gops_b200.create_pkg.create_alg import create_alg
    from test_oracle_rpi import rpi_kwargs
    torch.manual_seed(0)
    np.random.seed(0)
    alg = create_alg(**rpi_kwargs(reset_batch_size=B, sample_batch_size=B, max_newton_iteration=iters + 1))
    alg.networks.cuda()
    alg.local_update(None, 0)             # warm-up: module load, draw buffer, first launch (not timed)
    steps, times = [], []
    for it in range(1, iters + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        alg.local_update(None, it)        # ends in the iteration's device read
        times.append(time.perf_counter() - t0)
        steps.append(alg.num_update_value)
    total = sum(times)
    return dict(impl="gpu", batch=B, newton_iterations=iters, inner_steps=steps, inner_steps_per_s=sum(steps) / total,
                ms_per_newton_iteration=1e3 * total / iters, us_per_inner_step=1e6 * total / sum(steps))


def reference_leg(iters):
    from oracle import ref_shim
    from oracle.make_golden_rpi import kwargs
    if not ref_shim.available():
        return dict(impl="reference_cpu", error="reference not available (oracle/_ref not built)")
    ref_shim.install()
    from gops.create_pkg.create_alg import create_alg
    torch.manual_seed(0)
    np.random.seed(0)
    alg = create_alg(**kwargs())
    steps, times = [], []
    for it in range(iters):
        t0 = time.perf_counter()
        alg.local_update(None, it)
        times.append(time.perf_counter() - t0)
        steps.append(alg.num_update_value)
    total = sum(times)
    return dict(impl="reference_cpu", batch=64, newton_iterations=iters, inner_steps=steps, torch_threads=torch.get_num_threads(),
                inner_steps_per_s=sum(steps) / total, ms_per_newton_iteration=1e3 * total / iters,
                us_per_inner_step=1e6 * total / sum(steps))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=13)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--no_reference", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rpi: needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    res = [gpu_leg(a.iters, 64), gpu_leg(a.iters, 512)]
    if not a.no_reference:
        res.append(reference_leg(a.iters))
    res.append(dict(device=card[0] if card else torch.cuda.get_device_name(), cpu_count=os.cpu_count()))
    for r in res:
        print(json.dumps(r))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
