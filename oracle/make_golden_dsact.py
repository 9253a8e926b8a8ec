"""Generate tests/golden/dsact_idp.npz by running the UNMODIFIED reference's DSACT (GOPS @ /root/reference) on CPU.

TEST INFRASTRUCTURE.  Run in the build container only (`python oracle/make_golden_dsact.py`); it writes no other file.
DSACT.local_update (dsact.py:114-358): 4 updates, B = 128, [64,64,64] gelu nets, delay_update = 2, on a fixed synthetic
replay batch.  The reference draws its Gaussian noise from torch's global generator inside the update; the draws are
RECORDED (wrappers around torch.normal and torch.distributions.normal._standard_normal, as make_golden.run_dsac does --
instrumentation of this script, the reference is untouched).  Per update the reference draws [eps_new, eps_next, z(q1),
z(q2), z(q1_target), z(q2_target), z(policy-loss q1), z(policy-loss q2)]; only draws 0, 1, 4 and 5 reach a result and are
stored as eps_new / eps_next / z1_next / z2_next.  Also stored: the tb values (including the running `mean_std1` /
`mean_std2`, which are not in the state_dict), the gradients of q1 / q2 / policy / log_alpha and log_alpha after every
update.

The state_dicts are stored in the compact form oracle/dsact_oracle.expand_golden expands: the initial online nets (the
targets start as copies of them) and, per update, nothing more -- every post-update state_dict follows bit for bit from
the initial one and the recorded gradients through torch.optim.Adam and the reference's Polyak arithmetic.  This script
checks that expansion against the state_dicts the reference produced, key by key, before it writes the file, and stores a
per-key sum so that the expansion is checked again wherever it is loaded."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle import dsact_oracle as dto  # noqa: E402
from oracle import gops_oracle as orc  # noqa: E402
from oracle.make_golden import OUT, _np, _sd, base_kwargs  # noqa: E402


def run_dsact(name="dsact_idp", n_iter=4, B=128, hidden=(64, 64, 64)):
    from gops.create_pkg.create_alg import create_alg
    import torch.distributions.normal as tdn

    kw = base_kwargs("pyth_idpendulum", "DSACT", 6, 1, hidden, "gelu", "StochaPolicy",
                     value_func_name="ActionValueDistri", policy_act_distribution="TanhGaussDistribution",
                     value_learning_rate=dto.GOLDEN["lr_q"], policy_learning_rate=dto.GOLDEN["lr_policy"],
                     alpha_learning_rate=5e-3, gamma=0.99, tau=dto.GOLDEN["tau"], auto_alpha=True, alpha=0.2,
                     delay_update=dto.GOLDEN["delay_update"], policy_min_log_std=-20, policy_max_log_std=1,
                     value_hidden_sizes=list(hidden), policy_hidden_sizes=list(hidden))
    torch.manual_seed(778)
    alg = create_alg(**kw)
    g = torch.Generator().manual_seed(6)
    obs = orc.sample_inputs("pyth_idpendulum", B, 61)["obs"]
    data = {"obs": obs, "act": torch.rand(B, 1, generator=g) * 2 - 1, "rew": torch.randn(B, generator=g) * 3 + 5,
            "obs2": obs + 0.05 * torch.randn(B, 6, generator=g), "done": (torch.rand(B, generator=g) < 0.05).float()}
    rec = {"in_" + k: _np(v) for k, v in data.items()}
    full = {}
    for k, v in _sd(alg).items():
        full["init/" + k] = v
        if not k.split(".")[0].endswith("_target"):
            rec["init/" + k] = v
    noise = []
    o_sn, o_nm = tdn._standard_normal, torch.normal

    def sn(*a, **k):
        x = o_sn(*a, **k); noise.append(x.clone()); return x

    def nm(*a, **k):
        x = o_nm(*a, **k); noise.append(x.clone()); return x
    tdn._standard_normal, torch.normal = sn, nm
    try:
        torch.manual_seed(4243)
        for it in range(n_iter):
            noise.clear()
            tb = alg.local_update({k: v.clone() for k, v in data.items()}, it)
            assert len(noise) == 8, len(noise)
            for key, j in (("eps_new", 0), ("eps_next", 1), ("z1_next", 4), ("z2_next", 5)):
                rec[f"it{it}/{key}"] = _np(noise[j])
            for k, v in tb.items():
                if "Time" not in k:
                    rec[f"it{it}/tb/{k}"] = np.float64(v)
            for nm_ in ("policy", "q1", "q2"):
                for pn, p in getattr(alg.networks, nm_).named_parameters():
                    rec[f"it{it}/grad/{nm_}.{pn}"] = _np(p.grad).copy()
            rec[f"it{it}/grad/log_alpha"] = _np(alg.networks.log_alpha.grad).copy()
            for k, v in _sd(alg).items():
                full[f"it{it}/post/{k}"] = v
            rec[f"it{it}/post/log_alpha"] = full[f"it{it}/post/log_alpha"]
    finally:
        tdn._standard_normal, torch.normal = o_sn, o_nm
    for k, v in full.items():
        if "/post/" in k:
            rec[k.replace("/post/", "/post_sum/")] = np.float64(v.astype(np.float64).sum())
    expanded = dto.expand_golden(rec)
    for k, v in full.items():
        assert np.array_equal(expanded[k], v), k
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
    print(name, os.path.getsize(os.path.join(OUT, name + ".npz")), "bytes",
          {k: float(v) for k, v in rec.items() if "it0/tb/" in k})


if __name__ == "__main__":
    ref_shim.install()
    torch.set_num_threads(4)
    run_dsact()
