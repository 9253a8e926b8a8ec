"""DSAC on the layer-wise wgmma path (algorithm/dsac.py, csrc/dsac.cu, csrc/dense_tc.cu) against
(a) the unmodified reference: tests/golden/dsac_idp.npz -- four consecutive `local_update`s replaying the Gaussian noise the
    reference drew (eps_new / eps_next / z_next recorded by oracle/make_golden.py), scalars, gradients of q / policy /
    log_alpha, the Adam steps (delayed policy update), Polyak targets and the temperature;
(b) the CPU oracle (oracle/dsac_oracle.py) at the BASELINE configuration: [256,256,256] gelu nets, minibatch 8192.
Bars: scalars 1e-4 relative, gradients 2e-4 relative L2 (BF16x3 six-term forward, three-term gradient products)."""
import numpy as np
import pytest
import torch

from golden_util import load, rel_l2
from oracle import dsac_oracle as do

pytestmark = pytest.mark.gpu


def _kwargs(hidden):
    return dict(env_id="pyth_idpendulum", algorithm="DSAC", seed=0, trainer="off_serial_trainer", use_gpu=True,
                action_type="continu", obsv_dim=6, action_dim=1, action_high_limit=np.ones(1, np.float32),
                action_low_limit=-np.ones(1, np.float32), policy_func_name="StochaPolicy", policy_func_type="MLP",
                policy_hidden_sizes=list(hidden), policy_hidden_activation="gelu",
                policy_act_distribution="TanhGaussDistribution", policy_min_log_std=-20, policy_max_log_std=1,
                value_func_name="ActionValueDistri", value_func_type="MLP", value_hidden_sizes=list(hidden),
                value_hidden_activation="gelu", value_learning_rate=3e-4, policy_learning_rate=3e-4,
                alpha_learning_rate=5e-3, gamma=0.99, tau=0.005, auto_alpha=True, alpha=0.2, delay_update=2, TD_bound=10,
                bound=True)


def _grads(net):
    return [p.grad.detach().cpu().numpy() for p in net.parameters()]


def test_dsac_four_updates_follow_the_reference():
    from gops_b200.create_pkg.create_alg import create_alg
    rec = load("dsac_idp")
    alg = create_alg(**_kwargs((64, 64, 64)))
    alg.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("init/")})
    data = {k[3:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("in_")}
    n_it = 1 + max(int(k[2:k.index("/")]) for k in rec if k.startswith("it"))
    for it in range(n_it):
        if it > 0:        # continue from the reference's own weights so that errors do not compound
            alg.load_state_dict({k.split("/post/")[1]: torch.from_numpy(v) for k, v in rec.items()
                                 if k.startswith(f"it{it - 1}/post/")})
        alg.noise_override = {k: torch.from_numpy(rec[f"it{it}/{k}"]) for k in ("eps_new", "eps_next", "z_next")}
        tb = alg.local_update(data, it)
        for k in (k for k in rec if k.startswith(f"it{it}/tb/")):
            ref = float(rec[k])
            assert abs(tb[k.split("/tb/")[1]] - ref) <= 1e-4 * max(1.0, abs(ref)), (it, k, tb[k.split("/tb/")[1]], ref)
        for net in ("q", "policy"):
            mod = getattr(alg.networks, net)
            names = [f"it{it}/grad/{net}.{n}" for n, _ in mod.named_parameters()]
            err = rel_l2(_grads(mod), [rec[k] for k in names])
            assert err < 2e-4, (it, net, err)
        assert abs(alg.networks.alpha_optimizer.grad - float(rec[f"it{it}/grad/log_alpha"])) < 2e-5
        sd = alg.state_dict()
        # temperature (host-side scalar Adam) and Polyak targets after the (possibly delayed) update
        assert abs(float(sd["log_alpha"]) - float(rec[f"it{it}/post/log_alpha"])) < 2e-6, it
        lr = 3e-4
        for k in (k for k in rec if k.startswith(f"it{it}/post/") and k.endswith("weight")):
            got, want = sd[k.split("/post/")[1]].cpu().numpy(), rec[k]
            delta = np.abs(got - want)
            assert delta.max() <= 2.1 * lr, (it, k, delta.max())
            assert np.mean(delta <= 2e-2 * lr + 1e-7) > 0.97, (it, k)


def test_dsac_baseline_config_against_oracle():
    """BASELINE config 4: DSAC idpendulum, [256,256,256] gelu, minibatch 8192 drawn from the on-device replay buffer."""
    from gops_b200.create_pkg.create_alg import create_alg
    from gops_b200.trainer.device_buffer import DeviceReplayBuffer
    torch.manual_seed(1)
    alg = create_alg(**_kwargs((256, 256, 256)))
    B = 8192
    buf = DeviceReplayBuffer(6, 1, 1 << 16, device="cuda", seed=3)
    g = torch.Generator().manual_seed(9)
    obs = (torch.rand(1 << 15, 6, generator=g) * 2 - 1) * torch.tensor([5, 0.1, 0.1, 0.3, 0.3, 0.3])
    buf.add_batch({"obs": obs, "act": torch.rand(1 << 15, 1, generator=g) * 2 - 1, "rew": torch.randn(1 << 15, generator=g) * 3,
                   "obs2": obs + 0.05 * torch.randn(1 << 15, 6, generator=g),
                   "done": (torch.rand(1 << 15, generator=g) < 0.05).float()})
    assert len(buf) == 1 << 15
    batch = buf.sample_batch(B)
    assert all(v.is_cuda and v.shape[0] == B for v in batch.values())
    noise = {"eps_new": torch.randn(B, 1, generator=g), "eps_next": torch.randn(B, 1, generator=g),
             "z_next": torch.randn(B, generator=g)}
    alg.noise_override = noise
    nets = alg.networks
    lay = lambda mod, seq, grad: [(getattr(mod, seq)[j].weight.detach().cpu().clone().requires_grad_(grad),
                                   getattr(mod, seq)[j].bias.detach().cpu().clone().requires_grad_(grad)) for j in (0, 2, 4, 6)]
    pol, polT = lay(nets.policy, "policy", True), lay(nets.policy_target, "policy", False)
    q, qT = lay(nets.q, "q", True), lay(nets.q_target, "q", False)
    log_alpha = nets.log_alpha.detach().cpu().clone().requires_grad_(True)
    cpu = {k: v.cpu() for k, v in batch.items()}
    cpu["act"] = cpu["act"].reshape(B, 1)
    lq, lp, la, info = do.dsac_losses(pol, polT, q, qT, log_alpha, cpu, noise, gamma=0.99)
    gq = torch.autograd.grad(lq, [t for pair in q for t in pair])
    gp = torch.autograd.grad(lp, [t for pair in pol for t in pair])
    tb, _ = alg.get_remote_update_info(batch, 0)
    assert abs(tb["Loss/Actor loss-RL iter"] - lp.item()) <= 1e-4 * max(1.0, abs(lp.item()))
    assert abs(tb["Loss/Critic loss-RL iter"] - lq.item()) <= 1e-4 * max(1.0, abs(lq.item()))
    assert abs(tb["DSAC/critic_avg_q-RL iter"] - info["q"]) < 1e-5 and abs(tb["DSAC/entropy-RL iter"] - info["entropy"]) < 1e-4
    assert rel_l2(_grads(nets.q), [x.numpy() for x in gq]) < 2e-4
    assert rel_l2(_grads(nets.policy), [x.numpy() for x in gp]) < 2e-4
    # without injected noise the update draws its own on the device and still runs
    alg.noise_override = None
    tb2 = alg.local_update(batch, 1)
    assert np.isfinite(tb2["Loss/Actor loss-RL iter"])
