"""The UNMODIFIED reference's SAC update with given Gaussian noise (TEST INFRASTRUCTURE: only tests/ and oracle/ may
import this).

SAC.local_update (gops/algorithm/sac.py:108-263) runs as the reference ships it, through oracle/ref_shim.py.  Its only
random numbers are the two standard-normal tensors TanhGaussDistribution.rsample draws per update (eps_new for the
actor's action, then eps_next for the target action); `update` serves given tensors in their place by wrapping
torch.distributions.normal._standard_normal for the duration of the call.  The reference is already plain PyTorch, so
no separate restatement of SAC is kept.  Pinned against the recorded reference runs by tests/test_oracle_sac.py.

The recorded runs are stored compactly (`expand_golden` rebuilds them), and the shipped SAC checkpoint is not stored in
this repository at all: `copy_checkpoint` (called by __graft_entry__.build()) places the reference's own file next to
the reference copy in oracle/_ref, where `checkpoint_path` finds it on every machine the reference reaches."""
import filecmp
import hashlib
import os
import shutil

import numpy as np
import torch

from oracle import ref_shim


# the recorded runs of oracle/make_golden_sac.py: name -> (updates, batch, configuration overrides)
GOLDEN_CASES = {
    "sac_idp": (4, 128, dict(alpha_learning_rate=5e-3)),
    "sac_idp_fixed_alpha": (2, 128, dict(auto_alpha=False, alpha=0.1)),
}
# the shipped checkpoint (results/SAC/idpendulum, config.json): [256,256,256] relu nets
CKPT = dict(hidden=(256, 256, 256), act="relu", batch=256)
CKPT_INIT_STATE = [-1.0, 0.05, 0.05, 0.0, 0.1, 0.1]        # example_run/run_idp_sac_dsac.py init_state
CKPT_FILE = os.path.join("results", "SAC", "idpendulum", "apprfunc", "apprfunc_34500_opt.pkl")
_NETS = ("q1", "q2", "policy")


def checkpoint_path() -> str:
    """The shipped SAC checkpoint: in the reference tree, or in its copy oracle/_ref."""
    return os.path.join(ref_shim.REFERENCE_ROOT, CKPT_FILE)


def checkpoint_sha256(path=None) -> str:
    return hashlib.sha256(open(path or checkpoint_path(), "rb").read()).hexdigest()


def copy_checkpoint() -> bool:
    """Recipe for oracle/_ref: copy the reference's shipped SAC checkpoint byte for byte next to the reference copy
    that oracle/build_ref.py makes (a data file of the reference; oracle/_ref is git-ignored).  False when the
    reference tree is not here (the copy that travelled with the tree is used)."""
    from oracle import build_ref
    src, dst = os.path.join(build_ref.SRC, CKPT_FILE), os.path.join(build_ref.DST, CKPT_FILE)
    if not os.path.exists(src):
        return False
    if not (os.path.exists(dst) and filecmp.cmp(src, dst, shallow=False)):
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
    return True


def expand_golden(rec, kw):
    """The full record of a compact run of oracle/make_golden_sac.py: the initial target critics (copies of the online
    ones, as the reference's deepcopy makes them) and every post-update state_dict `it{k}/post/*`, rebuilt from the
    initial weights and the recorded gradients by the reference's own arithmetic (sac.py:243-263): torch.optim.Adam on
    q1, q2 and the policy, then Polyak  p_targ * (1 - tau) + (1 - polyak) * p  on the two critic targets.  log_alpha
    after each update is recorded as such.  The generator checks this rebuild bit for bit against the reference's
    state_dicts before it writes the file."""
    out = dict(rec)
    init = {k[5:]: v for k, v in rec.items() if k.startswith("init/")}
    for k in [k for k in init if k.split(".")[0] in ("q1", "q2")]:
        net = k.split(".")[0]
        init[net + "_target" + k[len(net):]] = init[k].copy()
    out.update({"init/" + k: v for k, v in init.items()})
    names = {net: [k for k in init if k.startswith(net + ".") and k.endswith(("weight", "bias"))] for net in _NETS}
    params = {net: [torch.nn.Parameter(torch.tensor(init[k])) for k in names[net]] for net in _NETS}
    targets = {net: [torch.tensor(init[net + "_target" + k[len(net):]]) for k in names[net]] for net in ("q1", "q2")}
    lr = {"q1": kw["q_learning_rate"], "q2": kw["q_learning_rate"], "policy": kw["policy_learning_rate"]}
    opts = {net: torch.optim.Adam(params[net], lr=lr[net]) for net in _NETS}
    polyak = 1 - kw["tau"]
    n_it = 1 + max(int(k[2:k.index("/")]) for k in rec if k.startswith("it"))
    for it in range(n_it):
        for net in _NETS:
            for p, k in zip(params[net], names[net]):
                p.grad = torch.tensor(rec[f"it{it}/grad/{k}"])
            opts[net].step()
        with torch.no_grad():
            for net in ("q1", "q2"):
                for t, p in zip(targets[net], params[net]):
                    t.mul_(polyak)
                    t.add_((1 - polyak) * p)
        post = {k: v for k, v in init.items() if k.endswith("_lim")}
        for net in _NETS:
            for k, p in zip(names[net], params[net]):
                post[k] = p.detach().numpy().copy()
        for net in ("q1", "q2"):
            for k, t in zip(names[net], targets[net]):
                post[net + "_target" + k[len(net):]] = t.numpy().copy()
        post["log_alpha"] = rec[f"it{it}/post/log_alpha"]
        out.update({f"it{it}/post/{k}": v for k, v in post.items()})
    return out


def kwargs(hidden=(64, 64, 64), act="gelu", **over):
    """A SAC configuration on pyth_idpendulum (results/SAC/idpendulum/config.json with the given nets)."""
    kw = dict(env_id="pyth_idpendulum", algorithm="SAC", seed=0, trainer="off_serial_trainer", cnn_shared=False,
              use_gpu=False, action_type="continu", obsv_dim=6, action_dim=1,
              action_high_limit=np.ones(1, np.float32), action_low_limit=-np.ones(1, np.float32),
              policy_func_name="StochaPolicy", policy_func_type="MLP", policy_hidden_sizes=list(hidden),
              policy_hidden_activation=act, policy_output_activation="linear",
              policy_act_distribution="TanhGaussDistribution", policy_min_log_std=-20, policy_max_log_std=1,
              value_func_name="ActionValue", value_func_type="MLP", value_hidden_sizes=list(hidden),
              value_hidden_activation=act, value_output_activation="linear", q_learning_rate=3e-4,
              value_learning_rate=3e-4, policy_learning_rate=3e-4, alpha_learning_rate=5e-5, gamma=0.99, tau=0.005,
              auto_alpha=True, alpha=0.2)
    kw.update(over)
    return kw


def create(kw, state_dict=None):
    """The reference's SAC from its own factory (create_alg.py:60-97), optionally loaded with a state_dict."""
    ref_shim.install()
    from gops.create_pkg.create_alg import create_alg
    alg = create_alg(**kw)
    if state_dict is not None:
        alg.load_state_dict({k: torch.as_tensor(np.asarray(v)) for k, v in state_dict.items()})
    return alg


def update(alg, data, eps_new, eps_next, iteration, remote=False):
    """One reference update with the given noise: local_update, or get_remote_update_info followed by remote_update
    (remote=True).  `data` is copied (the reference writes new_act / new_logp into its argument).  Returns the tb values
    (without the timing), the gradients it leaves in q1 / q2 / policy / log_alpha (`{net}.{param}` keys) and the
    post-update state_dict, as numpy arrays."""
    import torch.distributions.normal as tdn
    draws = [torch.as_tensor(eps_new, dtype=torch.float32), torch.as_tensor(eps_next, dtype=torch.float32)]
    served = []
    orig = tdn._standard_normal

    def given(shape, dtype, device):
        x = draws[len(served)]
        served.append(x)
        return x.reshape(shape).to(dtype=dtype, device=device).clone()
    tdn._standard_normal = given
    try:
        batch = {k: v.clone() for k, v in data.items()}
        if remote:
            tb, info = alg.get_remote_update_info(batch, iteration)
            alg.remote_update(info)
        else:
            tb = alg.local_update(batch, iteration)
    finally:
        tdn._standard_normal = orig
    assert len(served) == 2, len(served)
    nets = alg.networks
    grads = {f"{name}.{pn}": p.grad.detach().numpy().copy()
             for name in ("q1", "q2", "policy") for pn, p in getattr(nets, name).named_parameters()}
    if nets.log_alpha.grad is not None:
        grads["log_alpha"] = nets.log_alpha.grad.detach().numpy().copy()
    sd = {k: v.detach().numpy().copy() for k, v in alg.state_dict().items()}
    return {k: float(v) for k, v in tb.items() if "Time" not in k}, grads, sd
