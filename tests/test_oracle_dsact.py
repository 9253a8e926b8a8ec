"""CPU: pins oracle/dsact_oracle.py against the unmodified reference's DSACT.local_update (tests/golden/dsact_idp.npz, made
by oracle/make_golden_dsact.py with the reference's noise recorded): scalars, the running std means, gradients of
q1 / q2 / policy / log_alpha for four consecutive updates, each starting from the reference's own post-update weights
and running means."""
import torch

from golden_util import load, rel_l2
from oracle import dsact_oracle as dto


def _layers(rec, prefix, net, seq, grad):
    out, j = [], 0
    while f"{prefix}{net}.{seq}.{j}.weight" in rec:
        out.append((torch.tensor(rec[f"{prefix}{net}.{seq}.{j}.weight"]).requires_grad_(grad),
                    torch.tensor(rec[f"{prefix}{net}.{seq}.{j}.bias"]).requires_grad_(grad)))
        j += 2
    return out


def test_dsact_oracle_matches_reference():
    torch.set_num_threads(4)
    rec = dto.expand_golden(load("dsact_idp"), check_sums=True)
    data = {k[3:]: torch.tensor(v) for k, v in rec.items() if k.startswith("in_")}
    n_it = 1 + max(int(k[2:k.index("/")]) for k in rec if k.startswith("it"))
    assert n_it == 4
    for it in range(n_it):
        prefix = "init/" if it == 0 else f"it{it - 1}/post/"
        pol, polT = _layers(rec, prefix, "policy", "policy", True), _layers(rec, prefix, "policy_target", "policy", False)
        q1, q2 = _layers(rec, prefix, "q1", "q", True), _layers(rec, prefix, "q2", "q", True)
        q1T, q2T = _layers(rec, prefix, "q1_target", "q", False), _layers(rec, prefix, "q2_target", "q", False)
        log_alpha = torch.tensor(rec[prefix + "log_alpha"]).requires_grad_(True)
        ms = (None, None) if it == 0 else tuple(float(rec[f"it{it - 1}/tb/DSAC2/mean_std{i}"]) for i in (1, 2))
        noise = {k: torch.tensor(rec[f"it{it}/{k}"]) for k in ("eps_new", "eps_next", "z1_next", "z2_next")}
        lq, lp, la, info = dto.dsact_losses(pol, polT, q1, q2, q1T, q2T, log_alpha, data, noise, gamma=0.99, mean_std=ms)
        gq1 = torch.autograd.grad(lq, [t for pair in q1 for t in pair], retain_graph=True)
        gq2 = torch.autograd.grad(lq, [t for pair in q2 for t in pair])
        gp = torch.autograd.grad(lp, [t for pair in pol for t in pair])
        ga = torch.autograd.grad(la, [log_alpha])[0]
        tb = {k.split("/tb/")[1]: float(v) for k, v in rec.items() if k.startswith(f"it{it}/tb/")}
        assert abs(lp.item() - tb["Loss/Actor loss-RL iter"]) <= 2e-6 * max(1.0, abs(lp.item())), it
        assert abs(lq.item() - tb["Loss/Critic loss-RL iter"]) <= 1e-6 * max(1.0, abs(lq.item())), it
        for key in ("q1", "q2", "std1", "std2", "min_std1", "min_std2"):
            assert abs(info[key] - tb[f"DSAC2/critic_avg_{key}-RL iter"]) < 1e-6, (it, key)
        for i in (1, 2):
            assert abs(info[f"mean_std{i}"] - tb[f"DSAC2/mean_std{i}"]) < 1e-6, (it, i)
        assert abs(info["entropy"] - tb["DSAC2/entropy-RL iter"]) < 2e-6 and abs(info["alpha"] - tb["DSAC2/alpha-RL iter"]) < 1e-6
        assert abs(info["policy_mean"] - tb["DSAC2/policy_mean-RL iter"]) < 1e-6
        assert abs(info["policy_std"] - tb["DSAC2/policy_std-RL iter"]) < 1e-6
        for net, g, layers in (("q1", gq1, q1), ("q2", gq2, q2)):
            names = [f"it{it}/grad/{net}.q.{2 * j}.{w}" for j in range(len(layers)) for w in ("weight", "bias")]
            assert sorted(names) == sorted(k for k in rec if k.startswith(f"it{it}/grad/{net}."))
            assert rel_l2([x.numpy() for x in g], [rec[k] for k in names]) < 1e-5, (it, net)
        names_p = [f"it{it}/grad/policy.policy.{2 * j}.{w}" for j in range(len(pol)) for w in ("weight", "bias")]
        assert sorted(names_p) == sorted(k for k in rec if k.startswith(f"it{it}/grad/policy."))
        assert rel_l2([x.numpy() for x in gp], [rec[k] for k in names_p]) < 1e-5, it
        assert abs(float(ga) - float(rec[f"it{it}/grad/log_alpha"])) <= 1e-5 * max(1.0, abs(float(ga))), it
