"""Throughput of the batched policy inference (gops_b200_mlp_forward) on the two 64-wide CUDA paths:
GOPS_B200_INFER=mma (mma.sync 3xTF32) vs tc (wgmma 3xTF32).  Prints one JSON line per (mode, batch)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gops_b200.apprfunc.mlp import FiniteHorizonPolicy  # noqa: E402


def main():
    torch.manual_seed(0)
    obs_dim = int(os.environ.get("OBS_DIM", 6))
    net = FiniteHorizonPolicy(obs_dim=obs_dim, act_dim=1, hidden_sizes=(64, 64), hidden_activation="gelu",
                              output_activation="linear", action_distribution_cls=None,
                              act_high_lim=np.ones(1, np.float32), act_low_lim=-np.ones(1, np.float32)).cuda()
    for B in (1 << 14, 1 << 18, 1 << 22):
        obs = torch.randn(B, obs_dim, device="cuda")
        for mode in ("mma", "tc"):
            os.environ["GOPS_B200_INFER"] = mode
            for _ in range(3):
                net(obs, 3)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n = 20
            e0.record()
            for _ in range(n):
                net(obs, 3)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / n
            flop = 2.0 * B * (64 * (obs_dim + 1) + 64 * 64 + 64)
            print(json.dumps({"mode": mode, "batch": B, "ms": round(ms, 4), "samples_per_s": B / ms * 1e3,
                              "tflops": flop / ms / 1e9}))


if __name__ == "__main__":
    main()
