"""Time per update of DSAC and DSAC-T, and of a paired twin-critic forward + backward against two single-network ones,
at the BASELINE DSAC configuration: pyth_idpendulum, [256,256,256] gelu nets, minibatch 8192 from the on-device replay
buffer.  CUDA events around every timed call (each update ends in its scalar read-back), median of 20 after 3 warm-ups;
launches per call from gops_b200_launch_count.  Prints one JSON line per leg, then one with the device.

    python tools/bench_dsact.py"""
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
from gops_b200.ops.layerwise_mlp import LayerwiseMlp, LayerwiseMlpPair  # noqa: E402
from gops_b200.trainer.device_buffer import DeviceReplayBuffer  # noqa: E402

B, HIDDEN, WARMUP, REPS = 8192, [256, 256, 256], 3, 20


def kwargs(algorithm):
    return dict(env_id="pyth_idpendulum", algorithm=algorithm, seed=0, trainer="off_serial_trainer", use_gpu=True,
                action_type="continu", obsv_dim=6, action_dim=1, action_high_limit=np.ones(1, np.float32),
                action_low_limit=-np.ones(1, np.float32), policy_func_name="StochaPolicy", policy_func_type="MLP",
                policy_hidden_sizes=HIDDEN, policy_hidden_activation="gelu", policy_act_distribution="TanhGaussDistribution",
                policy_min_log_std=-20, policy_max_log_std=1, value_func_name="ActionValueDistri", value_func_type="MLP",
                value_hidden_sizes=HIDDEN, value_hidden_activation="gelu", value_learning_rate=3e-4,
                policy_learning_rate=3e-4, alpha_learning_rate=5e-5, gamma=0.99, tau=0.005, auto_alpha=True, alpha=0.2,
                delay_update=2, TD_bound=10, bound=True)


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


def report(leg, ms, launches, **extra):
    print(json.dumps({"leg": leg, "ms": round(ms, 4), "launches": launches, **extra}), flush=True)


def main():
    assert torch.cuda.is_available(), "bench_dsact needs a CUDA device"
    dev = torch.device("cuda")
    torch.manual_seed(0)
    buf = DeviceReplayBuffer(6, 1, 1 << 18, device=dev, seed=1)
    g = torch.Generator(device=dev).manual_seed(2)
    n = 1 << 16
    o = (torch.rand(n, 6, device=dev, generator=g) * 2 - 1) * torch.tensor([5, 0.1, 0.1, 0.3, 0.3, 0.3], device=dev)
    buf.add_batch({"obs": o, "act": torch.rand(n, 1, device=dev, generator=g) * 2 - 1,
                   "rew": torch.randn(n, device=dev, generator=g), "obs2": o + 0.01 * torch.randn(n, 6, device=dev, generator=g),
                   "done": (torch.rand(n, device=dev, generator=g) < 0.05).float()})
    for algorithm in ("DSAC", "DSACT"):
        alg = create_alg(**kwargs(algorithm))
        report(algorithm, *timed(lambda i: alg.local_update(buf.sample_batch(B), i)), unit="per update", batch=B)
        del alg
    # one twin-critic forward (train) + backward (weight gradients) on the critic input [obs | act]
    sizes = [7] + HIDDEN + [2]
    nets = [LayerwiseMlp(sizes, "gelu", max_batch=B) for _ in range(2)]
    for net in nets:
        net.pack((torch.randn(net.nparam, device=dev, generator=g) * 0.05).contiguous())
    pair = LayerwiseMlpPair(*nets)
    x = torch.randn(B, 7, device=dev, generator=g)
    dy = torch.randn(B, 2, device=dev, generator=g) / B
    grads = [torch.empty(net.nparam, device=dev) for net in nets]

    def two_single(_):
        for net, grad in zip(nets, grads):
            net.forward(x, slot=0, train=True)
            net.backward(dy, slot=0, grad=grad)

    def paired(_):
        pair.forward(x, slot=0, train=True)
        pair.backward(dy, dy, slot=0, grad_a=grads[0], grad_b=grads[1])
    for leg, fn in (("critics two single fwd+bwd", two_single), ("critics paired fwd+bwd", paired),
                    ("critics two single fwd+bwd (repeat)", two_single), ("critics paired fwd+bwd (repeat)", paired)):
        report(leg, *timed(fn), unit="per twin pass", batch=B)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit": power, "warmup": WARMUP, "reps": REPS,
                      "statistic": "median"}))


if __name__ == "__main__":
    main()
