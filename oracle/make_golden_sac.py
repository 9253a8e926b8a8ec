"""Generate tests/golden/sac_idp.npz, sac_idp_fixed_alpha.npz and ckpt_sac_idp.npz by running the UNMODIFIED
reference's SAC (GOPS @ /root/reference) on the CPU.

TEST INFRASTRUCTURE.  Run in the build container only (`python oracle/make_golden_sac.py`); it writes no other file.
SAC.local_update (sac.py:108-263) draws its Gaussian noise from torch's global generator inside the update: two draws,
eps_new then eps_next (asserted per update).  They are RECORDED by a wrapper around
torch.distributions.normal._standard_normal (instrumentation of this script, the reference is untouched), as
make_golden_dsact.py does.

  sac_idp / sac_idp_fixed_alpha (oracle/sac_ref.GOLDEN_CASES): [64,64,64] gelu nets on a fixed synthetic replay batch
      of 128; the inputs, the initial online nets and log_alpha, and per update the noise, the tb values, the gradients
      of q1 / q2 / policy (/ log_alpha with auto_alpha) and log_alpha after it.  The post-update state_dicts follow from
      these through torch.optim.Adam and the reference's Polyak arithmetic (oracle/sac_ref.expand_golden); this script
      checks that rebuild bit for bit against the reference's own state_dicts before it writes the file.
  ckpt_sac_idp (results/SAC/idpendulum/apprfunc/apprfunc_34500_opt.pkl, [256,256,256] relu): the checkpoint itself is
      the reference's file (sac_ref.copy_checkpoint places it in oracle/_ref); stored are its sha256, the 5-step closed
      loop of the mode action (hi - lo)/2 tanh(mean) + (hi + lo)/2 through the reference's
      create_env_model("pyth_idpendulum") from the example_run init state with q1 / q2 at every (state, action), and one
      update from the trained weights at B = 256 (the config's replay_batch_size) on transitions of that env model from
      random states and actions: inputs, noise, tb values, and the float64 sum and L2 norm of every gradient tensor."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle import gops_oracle as orc  # noqa: E402
from oracle import sac_ref  # noqa: E402
from oracle.make_golden import OUT, _np, _sd  # noqa: E402

CKPT = sac_ref.checkpoint_path()


def _batch(B, seed):
    g = torch.Generator().manual_seed(seed)
    obs = orc.sample_inputs("pyth_idpendulum", B, seed)["obs"]
    return {"obs": obs, "act": torch.rand(B, 1, generator=g) * 2 - 1, "rew": torch.randn(B, generator=g) * 3 + 5,
            "obs2": obs + 0.05 * torch.randn(B, 6, generator=g), "done": (torch.rand(B, generator=g) < 0.05).float()}


def _recorded_updates(alg, data, n_iter, rec, grad_summary=False):
    """n_iter reference updates drawing their own noise; records noise, tb and gradients (or, with grad_summary, the
    float64 sum and L2 norm of every gradient tensor)."""
    import torch.distributions.normal as tdn
    noise = []
    orig = tdn._standard_normal

    def sn(*a, **k):
        x = orig(*a, **k)
        noise.append(x.clone())
        return x
    tdn._standard_normal = sn
    try:
        for it in range(n_iter):
            noise.clear()
            tb = alg.local_update({k: v.clone() for k, v in data.items()}, it)
            assert len(noise) == 2, len(noise)
            rec[f"it{it}/eps_new"], rec[f"it{it}/eps_next"] = _np(noise[0]), _np(noise[1])
            for k, v in tb.items():
                if "Time" not in k:
                    rec[f"it{it}/tb/{k}"] = np.float64(v)
            for name in ("q1", "q2", "policy"):
                for pn, p in getattr(alg.networks, name).named_parameters():
                    g = _np(p.grad).copy()
                    if grad_summary:
                        rec[f"it{it}/grad_sum/{name}.{pn}"] = g.astype(np.float64).sum()
                        rec[f"it{it}/grad_norm/{name}.{pn}"] = np.linalg.norm(g.astype(np.float64))
                    else:
                        rec[f"it{it}/grad/{name}.{pn}"] = g
            if alg.auto_alpha:
                rec[f"it{it}/grad/log_alpha"] = _np(alg.networks.log_alpha.grad).copy()
            yield it
    finally:
        tdn._standard_normal = orig


def run_case(name):
    n_iter, B, over = sac_ref.GOLDEN_CASES[name]
    torch.manual_seed(779)
    kw = sac_ref.kwargs(**over)
    alg = sac_ref.create(kw)
    data = _batch(B, 62)
    rec = {"in_" + k: _np(v) for k, v in data.items()}
    init = _sd(alg)
    for k, v in init.items():
        if k.split(".")[0].endswith("_target"):
            assert np.array_equal(v, init[k.replace("_target", "", 1)]), k     # deepcopies of the online critics
        else:
            rec["init/" + k] = v
    full = {}
    torch.manual_seed(4244)
    for it in _recorded_updates(alg, data, n_iter, rec):
        full.update({f"it{it}/post/{k}": v for k, v in _sd(alg).items()})
        rec[f"it{it}/post/log_alpha"] = full[f"it{it}/post/log_alpha"]
    expanded = sac_ref.expand_golden(rec, kw)
    assert sorted(k for k in expanded if "/post/" in k) == sorted(full)
    for k, v in full.items():
        assert np.array_equal(expanded[k], v), k
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
    print(name, os.path.getsize(os.path.join(OUT, name + ".npz")), "bytes",
          {k: float(v) for k, v in rec.items() if "it0/tb/" in k})


def run_ckpt():
    from gops.create_pkg.create_env_model import create_env_model
    c = sac_ref.CKPT
    alg = sac_ref.create(sac_ref.kwargs(c["hidden"], c["act"]), torch.load(CKPT, map_location="cpu"))
    rec = {"ckpt_sha256": np.str_(sac_ref.checkpoint_sha256(CKPT))}
    nets = alg.networks
    pol = nets.policy
    env = create_env_model(env_id="pyth_idpendulum")
    o = torch.tensor([sac_ref.CKPT_INIT_STATE], dtype=torch.float32)
    states, acts, q1s, q2s = [], [], [], []
    with torch.no_grad():
        d, info = torch.zeros(1), {}
        for _ in range(5):
            mean = pol(o)[..., :1]
            a = (pol.act_high_lim - pol.act_low_lim) / 2 * torch.tanh(mean) + (pol.act_high_lim + pol.act_low_lim) / 2
            states.append(_np(o)[0])
            acts.append(_np(a)[0])
            q1s.append(float(nets.q1(o, a)))
            q2s.append(float(nets.q2(o, a)))
            o, r, d, info = env.forward(o, a, d, info)
    rec["closed_loop_states"], rec["closed_loop_actions"] = np.stack(states), np.stack(acts)
    rec["closed_loop_q1"], rec["closed_loop_q2"] = np.asarray(q1s, np.float32), np.asarray(q2s, np.float32)
    data = _batch(c["batch"], 63)
    with torch.no_grad():       # transitions of the env model itself, so that the trained critics' targets are meaningful
        data["obs2"], data["rew"], data["done"], _ = env.forward(data["obs"], data["act"], torch.zeros(c["batch"]), {})
    data["done"] = data["done"].float()
    rec.update({"in_" + k: _np(v) for k, v in data.items()})
    torch.manual_seed(4245)
    for _ in _recorded_updates(alg, data, 1, rec, grad_summary=True):
        pass
    np.savez_compressed(os.path.join(OUT, "ckpt_sac_idp.npz"), **rec)
    print("ckpt_sac_idp", os.path.getsize(os.path.join(OUT, "ckpt_sac_idp.npz")), "bytes", rec["closed_loop_actions"].ravel(),
          {k: float(v) for k, v in rec.items() if "it0/tb/" in k})


if __name__ == "__main__":
    ref_shim.install()
    torch.set_num_threads(4)
    for case in sac_ref.GOLDEN_CASES:
        run_case(case)
    run_ckpt()
