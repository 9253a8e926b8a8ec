"""CPU restatement of the DSAC-T update (TEST INFRASTRUCTURE: only tests/ may import this).

Follows gops/algorithm/dsact.py:162-329 in plain PyTorch (autograd) with the helpers of oracle/dsac_oracle.py (the
apprfuncs and TanhGaussDistribution.rsample) and the Gaussian noise passed in explicitly: eps_new for the actor's
action, eps_next for the target action, z1_next / z2_next for the samples of the two target critics (the reference
draws these, and four more that reach no result, from torch's global generator).  Pinned against the unmodified
reference by tests/test_oracle_dsact.py on tests/golden/dsact_idp.npz."""
import numpy as np
import torch

from oracle.dsac_oracle import policy_logits, q_head, rsample

BIAS = 0.1
# hyper-parameters of the recorded run (oracle/make_golden_dsact.py) that the expansion of its state_dicts depends on
GOLDEN = dict(lr_q=3e-4, lr_policy=3e-4, tau=0.005, delay_update=2)
_SEQ = {"q1": "q", "q2": "q", "policy": "policy"}


def expand_golden(rec, check_sums=False):
    """The full record of tests/golden/dsact_idp.npz: adds the initial target nets (copies of the online nets, as the
    reference's deepcopy makes them) and every post-update state_dict `it{k}/post/*`, rebuilt from the initial weights
    and the recorded gradients by the reference's own arithmetic (dsact.py:331-358): torch.optim.Adam on q1 and q2 every
    update, on the policy every `delay_update`-th, then Polyak  p_targ * (1 - tau) + tau * p  on the three targets.
    log_alpha after each update is recorded as such.  check_sums: compare each rebuilt tensor with the sum recorded
    from the reference's (the file's generator checks the rebuild bit for bit)."""
    out = dict(rec)
    init = {k[5:]: v for k, v in rec.items() if k.startswith("init/")}
    for k in list(init):
        net = k.split(".")[0]
        if net in _SEQ:
            init[net + "_target" + k[len(net):]] = init[k].copy()
    for k, v in init.items():
        out["init/" + k] = v

    def names(net):
        seq, j, res = _SEQ[net], 0, []
        while f"{net}.{seq}.{j}.weight" in init:
            res += [f"{net}.{seq}.{j}.weight", f"{net}.{seq}.{j}.bias"]
            j += 2
        return res
    params = {net: [torch.nn.Parameter(torch.tensor(init[k])) for k in names(net)] for net in _SEQ}
    targets = {net: [torch.tensor(init[net + "_target" + k[len(net):]]) for k in names(net)] for net in _SEQ}
    lr = {"q1": GOLDEN["lr_q"], "q2": GOLDEN["lr_q"], "policy": GOLDEN["lr_policy"]}
    opts = {net: torch.optim.Adam(params[net], lr=lr[net]) for net in _SEQ}
    polyak = 1 - GOLDEN["tau"]
    n_it = 1 + max(int(k[2:k.index("/")]) for k in rec if k.startswith("it"))
    for it in range(n_it):
        stepped = ("q1", "q2", "policy") if it % GOLDEN["delay_update"] == 0 else ("q1", "q2")
        for net in stepped:
            for p, k in zip(params[net], names(net)):
                p.grad = torch.tensor(rec[f"it{it}/grad/{k}"])
            opts[net].step()
        if it % GOLDEN["delay_update"] == 0:
            with torch.no_grad():
                for net in _SEQ:
                    for t, p in zip(targets[net], params[net]):
                        t.mul_(polyak)
                        t.add_((1 - polyak) * p)
        post = {k: v for k, v in init.items() if k.endswith("_lim")}
        for net in _SEQ:
            for k, p, t in zip(names(net), params[net], targets[net]):
                post[k] = p.detach().numpy().copy()
                post[net + "_target" + k[len(net):]] = t.numpy().copy()
        post["log_alpha"] = rec[f"it{it}/post/log_alpha"]
        for k, v in post.items():
            if check_sums:
                s, ref = float(v.astype(np.float64).sum()), float(rec[f"it{it}/post_sum/{k}"])
                assert abs(s - ref) <= 1e-5 * float(np.abs(v).astype(np.float64).sum()) + 1e-12, (it, k, s, ref)
            out[f"it{it}/post/{k}"] = v
    return out


def _target(rew, done, gamma, q_next, alpha, logp2):
    return rew + (1 - done) * gamma * (q_next - alpha * logp2)


def dsact_losses(policy, policy_target, q1, q2, q1_target, q2_target, log_alpha, data, noise, gamma, mean_std=(None, None),
                 tau_b=0.005, min_log_std=-20.0, max_log_std=1.0, target_entropy=-1.0, hi=None, lo=None, act="gelu"):
    """One DSACT.__compute_gradient (dsact.py:162-218): returns (loss_q, loss_policy, loss_alpha, info) whose autograd
    gradients are those the reference leaves in q1 / q2 / policy / log_alpha (critics frozen for the actor loss).
    `mean_std` holds the running means before this update (None = unset); info carries the updated ones."""
    obs, a, rew, obs2, done = data["obs"], data["act"], data["rew"], data["obs2"], data["done"]
    hi = torch.ones(a.shape[-1], dtype=obs.dtype) if hi is None else hi
    lo = -torch.ones(a.shape[-1], dtype=obs.dtype) if lo is None else lo
    alpha = log_alpha.detach().exp().item()
    logits = policy_logits(policy, obs, min_log_std, max_log_std, act)
    new_act, new_logp = rsample(logits, noise["eps_new"], hi, lo)
    with torch.no_grad():
        logits2 = policy_logits(policy_target, obs2, min_log_std, max_log_std, act)
        act2, logp2 = rsample(logits2, noise["eps_next"], hi, lo)
        samples = []
        for qt, z in ((q1_target, noise["z1_next"]), (q2_target, noise["z2_next"])):
            m, s = q_head(qt, obs2, act2, act)
            samples.append((m, m + torch.clamp(z, -3, 3) * s))
        (n1, s1), (n2, s2) = samples
        q_next = torch.min(n1, n2)
        q_next_sample = torch.where(n1 < n2, s1, s2)
        target = _target(rew, done, gamma, q_next, alpha, logp2)
        target_sample = _target(rew, done, gamma, q_next_sample, alpha, logp2)
    loss_q, info, new_ms = 0.0, {}, []
    for i, (q, ms) in enumerate(((q1, mean_std[0]), (q2, mean_std[1])), start=1):
        qm, qs = q_head(q, obs, a, act)
        m = torch.mean(qs.detach())
        ms = m if ms is None else (1 - tau_b) * torch.as_tensor(ms, dtype=torch.float32) + tau_b * m
        new_ms.append(ms)
        bound = 3 * ms
        target_b = qm.detach() + torch.clamp(target_sample - qm.detach(), -bound, bound)
        sd = torch.clamp(qs, min=0.0).detach()
        loss_q = loss_q + (ms ** 2 + BIAS) * torch.mean(
            -(target - qm).detach() / (sd ** 2 + BIAS) * qm
            - ((qm.detach() - target_b) ** 2 - sd ** 2) / (sd ** 3 + BIAS) * qs)
        info[f"q{i}"], info[f"std{i}"] = qm.detach().mean().item(), qs.detach().mean().item()
        info[f"min_std{i}"], info[f"mean_std{i}"] = qs.detach().min().item(), ms.item()
    frozen = lambda layers: [(w.detach(), b.detach()) for w, b in layers]
    qp1, _ = q_head(frozen(q1), obs, new_act, act)
    qp2, _ = q_head(frozen(q2), obs, new_act, act)
    loss_policy = (alpha * new_logp - torch.min(qp1, qp2)).mean()
    loss_alpha = -log_alpha * (new_logp.detach() + target_entropy).mean()
    info.update(entropy=-new_logp.detach().mean().item(), policy_mean=torch.tanh(logits[..., 0]).mean().item(),
                policy_std=logits[..., 1].mean().item(), alpha=alpha)
    return loss_q, loss_policy, loss_alpha, info
