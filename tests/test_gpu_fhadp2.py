"""FHADP2 / FiniteHorizonFullPolicy (open-loop policy, reference gops/algorithm/fhadp2.py, mlp.py:114-145) on the layer-wise
wgmma path: loss and gradient against an fp64 PyTorch restatement built from the oracle's env model (the rollout uses
the oracle's wrapped model step by step with the action sequence of ONE policy evaluation), the golden vectors of the
unmodified reference (tests/golden/fhadp2_idp.npz), and `forward_all_policy` inference."""
import numpy as np
import pytest
import torch

from golden_util import load, rel_l2
from oracle import gops_oracle as orc

pytestmark = pytest.mark.gpu


def _alg(env_id, obs_dim, act_dim, H, hid, act, seed, **extra):
    from gops_b200.create_pkg.create_alg import create_alg
    kw = dict(env_id=env_id, algorithm="FHADP2", seed=0, trainer="off_serial_trainer", use_gpu=True, action_type="continu",
              obsv_dim=obs_dim, action_dim=act_dim, action_high_limit=np.ones(act_dim, np.float32),
              action_low_limit=-np.ones(act_dim, np.float32), policy_func_name="FiniteHorizonFullPolicy",
              policy_func_type="MLP", policy_hidden_sizes=[hid, hid], policy_hidden_activation=act,
              policy_act_distribution="default", policy_learning_rate=1e-3, value_func_type="MLP", pre_horizon=H)
    kw.update(extra)
    torch.manual_seed(seed)
    return create_alg(**kw)


def _open_loop_loss(layers, act, env, data, H, act_dim, dtype):
    """fhadp2.py:98-121 with the oracle's model: a = policy.forward_all_policy(o); rollout under a[:, step]."""
    o, d, info = data["obs"], data["done"], data
    x = o
    for j, (w, b) in enumerate(layers):
        x = torch.nn.functional.linear(x, w, b)
        if j < len(layers) - 1:
            x = getattr(torch.nn.functional, act)(x)
    a_all = torch.tanh(x.reshape(o.shape[0], H, act_dim))        # act limits are +-1
    v = 0
    for step in range(H):
        o, r, d, info = env.forward(o, a_all[:, step], d, info)
        v = v + r if step == 0 else v + r * (1.0 ** step)
    return -v.mean()


@pytest.mark.parametrize("env_id,obs_dim,act_dim,H,hid,act,B", [
    ("pyth_idpendulum", 6, 1, 30, 64, "gelu", 1000),
    ("pyth_lq", 4, 2, 20, 256, "elu", 515),
])
def test_fhadp2_against_fp64(env_id, obs_dim, act_dim, H, hid, act, B):
    extra = dict(lq_config="s4a2") if env_id == "pyth_lq" else {}
    alg = _alg(env_id, obs_dim, act_dim, H, hid, act, seed=B, reward_scale=0.5, reward_shift=0.1, **extra)
    data = orc.sample_inputs(env_id, B, seed=B + 1, **extra)
    data["done"][::11] = 1.0
    pi = alg.networks.policy.pi
    layers = [(pi[j].weight.detach().cpu().double().requires_grad_(True), pi[j].bias.detach().cpu().double().requires_grad_(True))
              for j in (0, 2, 4)]
    env = orc.create_env_model(env_id, dtype=torch.float64, reward_scale=0.5, reward_shift=0.1, **extra)
    d64 = {k: v.double() for k, v in data.items()}
    loss = _open_loop_loss(layers, act, env, d64, H, act_dim, torch.float64)
    loss.backward()
    tb = alg.get_remote_update_info(data, 0)[0]
    torch.cuda.synchronize()
    assert alg.last_kernel_path() == "tc"
    got = tb["Loss/Actor loss-RL iter"]
    assert abs(got - loss.item()) <= 1e-4 * max(1.0, abs(loss.item())), (got, loss.item())
    got_g = [p.grad.detach().cpu().numpy() for p in alg.networks.policy.parameters()]
    ref_g = [t.grad.numpy() for pair in layers for t in pair]
    assert rel_l2(got_g, ref_g) < 2e-4
    # inference: the whole action sequence and its first element
    a_all = alg.networks.policy.forward_all_policy(data["obs"][:64])
    assert a_all.shape == (64, H, act_dim)
    with torch.no_grad():
        x = d64["obs"][:64]
        for j, (w, b) in enumerate(layers):
            x = torch.nn.functional.linear(x, w, b)
            if j < 2:
                x = getattr(torch.nn.functional, act)(x)
        want = torch.tanh(x.reshape(64, H, act_dim))
    np.testing.assert_allclose(a_all.numpy(), want.numpy(), rtol=0, atol=5e-6)
    np.testing.assert_allclose(alg.networks.policy(data["obs"][:64]).numpy(), want[:, 0].numpy(), rtol=0, atol=5e-6)


def test_fhadp2_golden_from_reference():
    rec = load("fhadp2_idp")
    H = int(rec["pre_horizon"])
    alg = _alg("pyth_idpendulum", 6, 1, H, 64, "gelu", seed=0, reward_scale=1.0)
    alg.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("init/")})
    data = {"obs": torch.from_numpy(rec["in_obs"]), "done": torch.from_numpy(rec["in_done"])}
    tb = alg.local_update(data, 0)
    ref_loss = float(rec["it0/tb/Loss/Actor loss-RL iter"])
    assert abs(tb["Loss/Actor loss-RL iter"] - ref_loss) <= 1e-4 * max(1.0, abs(ref_loss))
    gk = sorted(k for k in rec if k.startswith("it0/grad/policy."))
    named = dict(alg.networks.policy.named_parameters())
    assert rel_l2([named[k.split("/grad/policy.")[1]].grad.cpu().numpy() for k in gk], [rec[k] for k in gk]) < 2e-4
