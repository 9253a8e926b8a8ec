"""Time per update of SPIL on pyth_veh3dofconti_errcstr (value pass, device controller, policy pass, two Adam steps, two
Polyak averages) at B = 4096 and 2^16, next to INFADP on pyth_veh3dofconti (one PEV plus one PIM update) on the same
[64, 64] relu nets, forward_step 10, P = 10; and SPIL on pyth_mobilerobot with the shipped configuration ([64, 64] relu,
forward_step 25) at B = 1024 and 2^16, with the cost of its per-pass obstacle-noise draws timed on their own.  CUDA events around every timed call (each update ends in its scalar
read-back, loss_lag = 0), median of 20 after 3 warm-ups; launches per update from gops_b200_launch_count; fused-kernel
time per pass from the plans' own events (gops_b200_plan_enable_timing) in separate calls.  Prints one JSON line per leg,
then one with the device and its power limit.

    python tools/bench_spil.py"""
import ctypes
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gops_b200 import _lib  # noqa: E402
from gops_b200.create_pkg.create_alg import create_alg  # noqa: E402
from gops_b200.trainer.device_trainer import DeviceStateSampler  # noqa: E402

BATCHES, WARMUP, REPS = (4096, 1 << 16), 3, 20
ROBOT_BATCHES, ROBOT_H = (1024, 1 << 16), 25


def kwargs(algorithm, env_id):
    kw = dict(env_id=env_id, algorithm=algorithm, seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=46, action_dim=2, action_high_limit=np.ones(2, np.float32),
              action_low_limit=-np.ones(2, np.float32), policy_func_name="DetermPolicy", policy_func_type="MLP",
              policy_hidden_sizes=[64, 64], policy_hidden_activation="relu", policy_act_distribution="default",
              policy_learning_rate=1e-3, value_func_name="StateValue", value_func_type="MLP", value_hidden_sizes=[64, 64],
              value_hidden_activation="relu", value_learning_rate=1e-3, pre_horizon=10)
    if algorithm == "SPIL":
        kw.update(forward_step=10, constraint_dim=2, y_error_tol=0.1)
    return kw


def robot_kwargs():
    hi = np.array([0.4, np.pi / 3], np.float32)
    return dict(env_id="pyth_mobilerobot", algorithm="SPIL", seed=0, trainer="off_serial_trainer", use_gpu=True,
                action_type="continu", obsv_dim=13, action_dim=2, action_high_limit=hi, action_low_limit=-hi,
                policy_func_name="DetermPolicy", policy_func_type="MLP", policy_hidden_sizes=[64, 64],
                policy_hidden_activation="relu", policy_act_distribution="default", policy_learning_rate=3e-4,
                value_func_name="StateValue", value_func_type="MLP", value_hidden_sizes=[64, 64],
                value_hidden_activation="relu", value_learning_rate=2e-3, forward_step=ROBOT_H, constraint_dim=1)


def timed(step):
    """(median ms, launches per call) of step(i) over REPS calls after WARMUP."""
    L = _lib.lib()
    for i in range(WARMUP):
        step(i)
    torch.cuda.synchronize()
    ms, launches = [], []
    for i in range(REPS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        c0 = L.gops_b200_launch_count()
        e0.record()
        step(WARMUP + i)
        e1.record()
        launches.append(L.gops_b200_launch_count() - c0)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), statistics.median(launches)


def kernel_ms(alg, step):
    """Median fused-rollout kernel time of each of the algorithm's plans over REPS timed calls."""
    for plan in alg._plans.values():
        _lib.check(_lib.lib().gops_b200_plan_enable_timing(plan.handle, 1))
    per = {}
    for i in range(REPS):
        step(i)
        for (kind, _, _), plan in alg._plans.items():
            ms = ctypes.c_float()
            _lib.check(_lib.lib().gops_b200_plan_last_kernel_ms(plan.handle, ctypes.byref(ms)))
            per.setdefault(kind, []).append(ms.value)
    for plan in alg._plans.values():
        _lib.check(_lib.lib().gops_b200_plan_enable_timing(plan.handle, 0))
    names = {_lib.ALG_FHADP: "policy pass", _lib.ALG_INFADP_POLICY: "PIM", _lib.ALG_INFADP_VALUE: "value pass"}
    return {names[k]: round(statistics.median(v), 4) for k, v in per.items()}


def report(leg, ms, launches, **extra):
    print(json.dumps({"leg": leg, "ms": round(ms, 4), "launches": launches, **extra}), flush=True)


def main():
    assert torch.cuda.is_available(), "bench_spil needs a CUDA device"
    for B in BATCHES:
        torch.manual_seed(0)
        data = DeviceStateSampler("pyth_veh3dofconti_errcstr", "cuda", 1, pre_horizon=10).sample(B)
        spil = create_alg(**kwargs("SPIL", "pyth_veh3dofconti_errcstr"))
        report("SPIL", *timed(lambda i: spil.local_update(data, i)), unit="per update", batch=B,
               kernel_ms=kernel_ms(spil, lambda i: spil.local_update(data, i)))
        del spil
        infadp = create_alg(**kwargs("INFADP", "pyth_veh3dofconti"))
        # one PEV and one PIM update (iterations 2i and 2i + 1)
        two = lambda i: (infadp.local_update(data, 2 * i), infadp.local_update(data, 2 * i + 1))
        report("INFADP PEV+PIM", *timed(two), unit="per PEV+PIM pair", batch=B, kernel_ms=kernel_ms(infadp, two))
        del infadp
    for B in ROBOT_BATCHES:
        torch.manual_seed(0)
        data = DeviceStateSampler("pyth_mobilerobot", "cuda", 1).sample(B)
        spil = create_alg(**robot_kwargs())
        model = spil.envmodel.unwrapped
        # one pass's draws: torch.randn and the std scaling, ROBOT_H * B * 2 floats (8 bytes per sample and step)
        dev = spil._device()     # the device (and so the generator) the update's own draws use
        draw_ms, _ = timed(lambda i: model.draw_noise((ROBOT_H, B, 2), dev))
        report("SPIL mobilerobot", *timed(lambda i: spil.local_update(data, i)), unit="per update", batch=B,
               kernel_ms=kernel_ms(spil, lambda i: spil.local_update(data, i)), noise_draw_ms_per_pass=round(draw_ms, 4),
               noise_bytes_per_pass=ROBOT_H * B * 2 * 4)
        del spil
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "unknown"
    print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit": q, "warmup": WARMUP, "reps": REPS,
                      "statistic": "median"}))


if __name__ == "__main__":
    main()
