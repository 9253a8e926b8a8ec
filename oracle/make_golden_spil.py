"""Generate tests/golden/spil_*.npz by running the UNMODIFIED reference's SPIL (GOPS @ /root/reference) on CPU.

TEST INFRASTRUCTURE.  Run in the build container only (`python oracle/make_golden_spil.py`); it writes no other file.
SPIL.local_update (spil.py:126-270) on pyth_veh3dofconti_errcstr: B = 160 with every ninth sample done, DetermPolicy and
StateValue [64, 64] relu, forward_step 10, 4 consecutive updates on one batch.  Stored per update: the tb values, the
gradients of v and policy, the post-update state_dict and the controller's safe_prob / lam / delta_i.

Two settings of the error tolerances: "near" keeps the safe probability within 0.1 of the 0.97 threshold (the
proportional-integral branch), "far" keeps it more than 0.2 below (the separated integral).  Safety is a discrete count,
so the script records every constraint value the reference's rollouts see and refuses to write a file in which one lies
within 1e-4 of 0 (where fp32 round-off could flip a count)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle import gops_oracle as orc  # noqa: E402
from oracle.make_golden import OUT, _np, _sd, base_kwargs, flat_inputs, to_ref_data  # noqa: E402

SETTINGS = {"spil_near": dict(y_error_tol=3.0, u_error_tol=2.3, seed=81),
            "spil_far": dict(y_error_tol=0.9, u_error_tol=1.6, seed=82)}
B, N_UPDATES, FORWARD_STEP = 160, 4, 10
C_MIN = 1e-4


def kwargs_of(setting):
    s = SETTINGS[setting]
    return base_kwargs("pyth_veh3dofconti_errcstr", "SPIL", 46, 2, (64, 64), "relu", "DetermPolicy", pre_horizon=10,
                       forward_step=FORWARD_STEP, constraint_dim=2, y_error_tol=s["y_error_tol"],
                       u_error_tol=s["u_error_tol"], gamma=0.99, tau=0.005)


def batch_of(setting):
    d = orc.sample_inputs("pyth_veh3dofconti", B, SETTINGS[setting]["seed"], pre_horizon=10)
    d["done"][::9] = 1.0
    return d


def run_spil(setting, write=True):
    from gops.create_pkg.create_alg import create_alg

    torch.manual_seed(1234)
    alg = create_alg(**kwargs_of(setting))
    data = batch_of(setting)
    rec = flat_inputs("pyth_veh3dofconti", data)
    for k, v in _sd(alg).items():
        rec["init/" + k] = v
    seen = []
    forward = alg.envmodel.forward

    def recording_forward(o, a, d, info):           # instrumentation of this script: the reference is untouched
        out = forward(o, a, d, info)
        seen.append(out[3]["constraint"].detach().abs().min().item())
        return out
    alg.envmodel.forward = recording_forward
    ref_data = to_ref_data("pyth_veh3dofconti", data)
    ref_data["constraint"] = torch.zeros(B, 2)
    for it in range(N_UPDATES):
        tb = alg.local_update({k: v.clone() for k, v in ref_data.items()}, it)
        for k, v in tb.items():
            if "Time" not in k:
                rec[f"it{it}/tb/{k}"] = np.float64(v)
        for nm in ("policy", "v"):
            for pn, p in getattr(alg.networks, nm).named_parameters():
                rec[f"it{it}/grad/{nm}.{pn}"] = _np(p.grad).copy()
        for k, v in _sd(alg).items():
            rec[f"it{it}/post/{k}"] = v
        rec[f"it{it}/safe_prob"] = np.asarray(alg.safe_prob, dtype=np.float32)
        rec[f"it{it}/lam"] = np.asarray(alg.lam, dtype=np.float64)
        rec[f"it{it}/delta_i"] = np.asarray(alg.delta_i, dtype=np.float64)
    assert min(seen) >= C_MIN, f"{setting}: a constraint value lies within {C_MIN} of 0 ({min(seen):.3g})"
    print(setting, "min |c|", min(seen), {k: rec[k].tolist() for k in rec if k.endswith(("safe_prob", "lam"))})
    if write:
        np.savez_compressed(os.path.join(OUT, setting + ".npz"), **rec)
    return rec


if __name__ == "__main__":
    ref_shim.install()
    torch.set_num_threads(4)
    for name in SETTINGS:
        run_spil(name, write="--dry" not in sys.argv)
