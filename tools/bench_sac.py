"""Time per SAC update at the shipped configuration (results/SAC/idpendulum/config.json): pyth_idpendulum,
[256,256,256] relu nets, minibatches from the on-device replay buffer, at B = 256 (the config's replay_batch_size) and
B = 8192, with DSAC-T at 8192 in the same run as the neighbour.  CUDA events around every update (each ends in its
scalar read-back), median of 20 after 3 warm-ups; launches per update from gops_b200_launch_count.  Prints one JSON line
per leg, then one with the device and its power limit.

    python tools/bench_sac.py [--reference]

--reference adds the unmodified reference's SAC (oracle/_ref, oracle/build_ref.py) in PyTorch eager on the same GPU,
labelled as such; it is not part of this library."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gops_b200.create_pkg.create_alg import create_alg  # noqa: E402
from gops_b200.trainer.device_buffer import DeviceReplayBuffer  # noqa: E402
from tools.bench_dsact import kwargs as dsact_kwargs, report, timed  # noqa: E402

HIDDEN = [256, 256, 256]


def sac_kwargs():
    return dict(env_id="pyth_idpendulum", algorithm="SAC", seed=0, trainer="off_serial_trainer", use_gpu=True,
                action_type="continu", obsv_dim=6, action_dim=1, action_high_limit=np.ones(1, np.float32),
                action_low_limit=-np.ones(1, np.float32), policy_func_name="StochaPolicy", policy_func_type="MLP",
                policy_hidden_sizes=HIDDEN, policy_hidden_activation="relu", policy_output_activation="linear",
                policy_act_distribution="TanhGaussDistribution", policy_min_log_std=-20, policy_max_log_std=1,
                value_func_name="ActionValue", value_func_type="MLP", value_hidden_sizes=HIDDEN,
                value_hidden_activation="relu", value_output_activation="linear", q_learning_rate=3e-4,
                value_learning_rate=3e-4, policy_learning_rate=3e-4, alpha_learning_rate=5e-5)


def reference_sac(buf, B, dev):
    """The unmodified reference's SAC.local_update in PyTorch eager on `dev` (not this library)."""
    from oracle import ref_runner
    alg = ref_runner.create_reference_alg(dict(sac_kwargs(), use_gpu=True), device=dev)

    def step(i):
        alg.local_update(buf.sample_batch(B), i)
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", action="store_true", help="also time the unmodified reference's SAC in eager mode")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sac needs a CUDA device"
    dev = torch.device("cuda")
    torch.manual_seed(0)
    buf = DeviceReplayBuffer(6, 1, 1 << 18, device=dev, seed=1)
    g = torch.Generator(device=dev).manual_seed(2)
    n = 1 << 16
    o = (torch.rand(n, 6, device=dev, generator=g) * 2 - 1) * torch.tensor([5, 0.1, 0.1, 0.3, 0.3, 0.3], device=dev)
    buf.add_batch({"obs": o, "act": torch.rand(n, 1, device=dev, generator=g) * 2 - 1,
                   "rew": torch.randn(n, device=dev, generator=g), "obs2": o + 0.01 * torch.randn(n, 6, device=dev, generator=g),
                   "done": (torch.rand(n, device=dev, generator=g) < 0.05).float()})
    for algorithm, kw, B in (("SAC", sac_kwargs(), 256), ("SAC", sac_kwargs(), 8192), ("DSACT", dsact_kwargs("DSACT"), 8192)):
        alg = create_alg(**kw)
        report(algorithm, *timed(lambda i: alg.local_update(buf.sample_batch(B), i)), unit="per update", batch=B,
               nets=f"{HIDDEN} {kw['value_hidden_activation']}")
        del alg
    if args.reference:
        for B in (256, 8192):
            ms, _ = timed(reference_sac(buf, B, dev))
            report("reference SAC, PyTorch eager (not this library)", ms, None, unit="per update", batch=B)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit": power, "warmup": 3, "reps": 20,
                      "statistic": "median"}))


if __name__ == "__main__":
    main()
