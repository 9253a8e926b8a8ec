"""DSAC-T on paired layer-wise wgmma passes (algorithm/dsact.py, csrc/dsact.cu, csrc/dense_tc.cu mlpnet_pair_*) against
(a) the unmodified reference: tests/golden/dsact_idp.npz -- four consecutive `local_update`s replaying the Gaussian noise
    the reference drew (eps_new / eps_next / z1_next / z2_next recorded by oracle/make_golden_dsact.py) and resuming
    each from the reference's weights and running std means: scalars, gradients of q1 / q2 / policy / log_alpha, the
    Adam steps (delayed policy update), Polyak targets and the temperature;
(b) the CPU oracle (oracle/dsact_oracle.py) at the BASELINE DSAC size: [256,256,256] gelu nets, minibatch 8192 from the
    on-device replay buffer, including the first Adam / Polyak step;
and the paired passes themselves: bit-identical to two single-network passes, the launches of one, mismatches refused.
Bars: scalars 1e-4 relative, gradients 2e-4 relative L2 (BF16x3 six-term forward, three-term gradient products)."""
import numpy as np
import pytest
import torch

from golden_util import load, rel_l2
from oracle import dsact_oracle as dto

pytestmark = pytest.mark.gpu

LR_Q, LR_PI, LR_ALPHA, TAU = 3e-4, 3e-4, 5e-3, 0.005


def _kwargs(hidden):
    return dict(env_id="pyth_idpendulum", algorithm="DSACT", seed=0, trainer="off_serial_trainer", use_gpu=True,
                action_type="continu", obsv_dim=6, action_dim=1, action_high_limit=np.ones(1, np.float32),
                action_low_limit=-np.ones(1, np.float32), policy_func_name="StochaPolicy", policy_func_type="MLP",
                policy_hidden_sizes=list(hidden), policy_hidden_activation="gelu",
                policy_act_distribution="TanhGaussDistribution", policy_min_log_std=-20, policy_max_log_std=1,
                value_func_name="ActionValueDistri", value_func_type="MLP", value_hidden_sizes=list(hidden),
                value_hidden_activation="gelu", value_learning_rate=LR_Q, policy_learning_rate=LR_PI,
                alpha_learning_rate=LR_ALPHA, gamma=0.99, tau=TAU, auto_alpha=True, alpha=0.2, delay_update=2)


def _grads(net):
    return [p.grad.detach().cpu().numpy() for p in net.parameters()]


def _check_weights(sd, want, lr_of, tag):
    """Adam moves every weight by at most ~lr on its first steps: the update must land within 2.1 lr of the expected
    weights everywhere and within 2 % of lr on nearly all of them (a different sign or scale of the step shows)."""
    for k, w in want.items():
        if not k.endswith("weight"):
            continue
        lr = lr_of(k)
        delta = np.abs(sd[k].cpu().numpy() - w)
        assert delta.max() <= 2.1 * lr, (tag, k, delta.max())
        assert np.mean(delta <= 2e-2 * lr + 1e-7) > 0.97, (tag, k)


def _lr_of(k):
    return LR_PI if k.startswith("policy") else LR_Q


def test_dsact_four_updates_follow_the_reference():
    from gops_b200.create_pkg.create_alg import create_alg
    rec = dto.expand_golden(load("dsact_idp"), check_sums=True)
    alg = create_alg(**_kwargs((64, 64, 64)))
    alg.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("init/")})
    data = {k[3:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("in_")}
    n_it = 1 + max(int(k[2:k.index("/")]) for k in rec if k.startswith("it"))
    assert n_it == 4 and alg.mean_std1 is None and alg.mean_std2 is None
    for it in range(n_it):
        if it > 0:        # continue from the reference's own weights and running means so that errors do not compound
            alg.load_state_dict({k.split("/post/")[1]: torch.from_numpy(v) for k, v in rec.items()
                                 if k.startswith(f"it{it - 1}/post/")})
            alg.mean_std1 = float(rec[f"it{it - 1}/tb/DSAC2/mean_std1"])
            alg.mean_std2 = float(rec[f"it{it - 1}/tb/DSAC2/mean_std2"])
        alg.noise_override = {k: torch.from_numpy(rec[f"it{it}/{k}"]) for k in ("eps_new", "eps_next", "z1_next", "z2_next")}
        tb = alg.local_update(data, it)
        keys = [k for k in rec if k.startswith(f"it{it}/tb/")]
        assert len(keys) == 14
        for k in keys:
            ref, got = float(rec[k]), tb[k.split("/tb/")[1]]
            assert abs(got - ref) <= 1e-4 * max(1.0, abs(ref)), (it, k, got, ref)
        assert abs(alg.mean_std1 - float(rec[f"it{it}/tb/DSAC2/mean_std1"])) <= 1e-4 * max(1.0, alg.mean_std1)
        for net in ("q1", "q2", "policy"):
            mod = getattr(alg.networks, net)
            names = [f"it{it}/grad/{net}.{n}" for n, _ in mod.named_parameters()]
            err = rel_l2(_grads(mod), [rec[k] for k in names])
            assert err < 2e-4, (it, net, err)
        assert abs(alg.networks.alpha_optimizer.grad - float(rec[f"it{it}/grad/log_alpha"])) < 2e-5
        sd = alg.state_dict()
        assert abs(float(sd["log_alpha"]) - float(rec[f"it{it}/post/log_alpha"])) < 2e-6, it
        _check_weights(sd, {k.split("/post/")[1]: v for k, v in rec.items() if k.startswith(f"it{it}/post/")}, _lr_of,
                       it)


def test_dsact_state_dict_round_trips_into_the_reference_keys():
    from gops_b200.create_pkg.create_alg import create_alg
    rec = dto.expand_golden(load("dsact_idp"), check_sums=True)
    init = {k[5:]: v for k, v in rec.items() if k.startswith("init/")}
    alg = create_alg(**_kwargs((64, 64, 64)))
    assert set(alg.state_dict()) == set(init)
    alg.load_state_dict({k: torch.from_numpy(v) for k, v in init.items()})
    sd = alg.state_dict()
    for k, v in init.items():
        assert np.array_equal(sd[k].cpu().numpy(), v), k
    assert alg.adjustable_parameters == ("gamma", "tau", "auto_alpha", "alpha", "delay_update")


def _layers(mod, seq, grad):
    return [(getattr(mod, seq)[j].weight.detach().cpu().clone().requires_grad_(grad),
             getattr(mod, seq)[j].bias.detach().cpu().clone().requires_grad_(grad)) for j in (0, 2, 4, 6)]


def test_dsact_baseline_config_against_oracle():
    """BASELINE DSAC size: [256,256,256] gelu, minibatch 8192 drawn from the on-device replay buffer."""
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
    batch = buf.sample_batch(B)
    assert all(v.is_cuda and v.shape[0] == B for v in batch.values())
    noise = {"eps_new": torch.randn(B, 1, generator=g), "eps_next": torch.randn(B, 1, generator=g),
             "z1_next": torch.randn(B, generator=g), "z2_next": torch.randn(B, generator=g)}
    alg.noise_override = noise
    nets = alg.networks
    pol, polT = _layers(nets.policy, "policy", True), _layers(nets.policy_target, "policy", False)
    q1, q2 = _layers(nets.q1, "q", True), _layers(nets.q2, "q", True)
    q1T, q2T = _layers(nets.q1_target, "q", False), _layers(nets.q2_target, "q", False)
    log_alpha = nets.log_alpha.detach().cpu().clone().requires_grad_(True)
    # a resumed running mean: the EMA branch of the critic loss
    ms = (0.6, 0.75)
    alg.mean_std1, alg.mean_std2 = ms
    cpu = {k: v.cpu() for k, v in batch.items()}
    cpu["act"] = cpu["act"].reshape(B, 1)
    lq, lp, la, info = dto.dsact_losses(pol, polT, q1, q2, q1T, q2T, log_alpha, cpu, noise, gamma=0.99, mean_std=ms)
    flat = lambda layers: [t for pair in layers for t in pair]
    gq1 = torch.autograd.grad(lq, flat(q1), retain_graph=True)
    gq2 = torch.autograd.grad(lq, flat(q2))
    gp = torch.autograd.grad(lp, flat(pol))
    ga = torch.autograd.grad(la, [log_alpha])[0]
    tb, upd = alg.get_remote_update_info(batch, 0)
    close = lambda got, want: abs(got - want) <= 1e-4 * max(1.0, abs(want))
    assert close(tb["Loss/Actor loss-RL iter"], lp.item()) and close(tb["Loss/Critic loss-RL iter"], lq.item())
    for key in ("q1", "q2", "std1", "std2", "min_std1", "min_std2"):
        assert close(tb[f"DSAC2/critic_avg_{key}-RL iter"], info[key]), key
    for i in (1, 2):
        assert close(tb[f"DSAC2/mean_std{i}"], info[f"mean_std{i}"]), i
    assert close(tb["DSAC2/entropy-RL iter"], info["entropy"]) and close(tb["DSAC2/policy_mean-RL iter"], info["policy_mean"])
    assert close(tb["DSAC2/policy_std-RL iter"], info["policy_std"])
    for net, want in (("q1", gq1), ("q2", gq2), ("policy", gp)):
        assert rel_l2(_grads(getattr(nets, net)), [x.numpy() for x in want]) < 2e-4, net
    assert abs(upd["log_alpha_grad"] - float(ga)) < 2e-5
    assert sorted(upd) == ["iteration", "log_alpha_grad", "policy_grad", "q1_grad", "q2_grad"]
    # the first update (iteration 0: critics, delayed policy and temperature steps, Polyak) against torch.optim.Adam
    want = {}
    for name, layers, grads, lr in (("q1", q1, gq1, LR_Q), ("q2", q2, gq2, LR_Q), ("policy", pol, gp, LR_PI)):
        params = [t.detach().clone().requires_grad_(True) for t in flat(layers)]
        opt = torch.optim.Adam(params, lr=lr)
        for p, gr in zip(params, grads):
            p.grad = gr
        opt.step()
        seq = "policy" if name == "policy" else "q"
        for j, p in enumerate(params):
            want[f"{name}.{seq}.{2 * (j // 2)}.{('weight', 'bias')[j % 2]}"] = p.detach().numpy()
    for name, tgt, src in (("q1_target", q1T, "q1"), ("q2_target", q2T, "q2"), ("policy_target", polT, "policy")):
        seq = "policy" if src == "policy" else "q"
        for j, (w, _) in enumerate(tgt):
            want[f"{name}.{seq}.{2 * j}.weight"] = ((1 - TAU) * w + TAU * torch.from_numpy(want[f"{src}.{seq}.{2 * j}.weight"])).numpy()
    la_p = log_alpha.detach().clone().requires_grad_(True)
    opt = torch.optim.Adam([la_p], lr=LR_ALPHA)
    la_p.grad = ga.reshape(())
    opt.step()
    alg.remote_update(upd)
    sd = alg.state_dict()
    assert abs(float(sd["log_alpha"]) - float(la_p.detach())) < 2e-6
    _check_weights(sd, want, _lr_of, "baseline")


def test_dsact_runs_without_injected_noise():
    from gops_b200.create_pkg.create_alg import create_alg
    torch.manual_seed(2)
    alg = create_alg(**_kwargs((64, 64, 64)))
    B = 1000
    g = torch.Generator().manual_seed(4)
    obs = torch.randn(B, 6, generator=g) * 0.3
    data = {"obs": obs.cuda(), "act": (torch.rand(B, 1, generator=g) * 2 - 1).cuda(), "rew": torch.randn(B, generator=g).cuda(),
            "obs2": (obs + 0.05 * torch.randn(B, 6, generator=g)).cuda(), "done": torch.zeros(B).cuda()}
    for it in range(3):
        tb = alg.local_update(data, it)
        vals = [v for k, v in tb.items() if "Time" not in k]
        assert len(vals) == 14 and all(np.isfinite(v) for v in vals), tb
    assert alg.mean_std1 is not None and np.isfinite(alg.mean_std1) and np.isfinite(alg.mean_std2)


# ---------------------------------------------------------------------------------------------------- paired passes
def _net_pair(sizes, max_batch, seed):
    from gops_b200.ops.layerwise_mlp import LayerwiseMlp, LayerwiseMlpPair
    g = torch.Generator().manual_seed(seed)
    nets, params = [], []
    for _ in range(2):
        n = LayerwiseMlp(sizes, "gelu", max_batch=max_batch, slots=2)
        p = (torch.randn(n.nparam, generator=g) * 0.1).cuda()
        n.pack(p)
        nets.append(n)
        params.append(p)
    return nets, params, LayerwiseMlpPair(*nets)


@pytest.mark.parametrize("hidden", [(256, 256, 256), (64, 64, 64)])
def test_pair_passes_equal_two_single_passes(hidden):
    sizes = [7, *hidden, 2]
    B = 1000                                  # not a multiple of the 128-row tile
    (a, b), params, pair = _net_pair(sizes, 1024, 11)
    g = torch.Generator().manual_seed(12)
    xw = torch.randn(B, 9, generator=g).cuda()
    x = xw[:, :7]                             # a strided input (row stride 9), as the critics read [obs | act] rows
    dya, dyb = torch.randn(B, 2, generator=g).cuda(), torch.randn(B, 2, generator=g).cuda()
    single = {}
    for name, net, dy in (("a", a, dya), ("b", b, dyb)):
        grad = torch.full((net.nparam,), 0.5, device="cuda")
        y = net.forward(x, slot=1, train=True)
        dx = net.backward(dy, slot=1, grad=grad, accumulate=True, want_dx=True)
        single[name] = (y, grad, dx)
    ga = torch.full((a.nparam,), 0.5, device="cuda")
    gb = torch.full((b.nparam,), 0.5, device="cuda")
    ya, yb = pair.forward(x, slot=1, train=True)
    dxa, dxb = pair.backward(dya, dyb, slot=1, grad_a=ga, grad_b=gb, accumulate=True, want_dx=True)
    torch.cuda.synchronize()
    for got, want in zip((ya, ga, dxa), single["a"]):
        assert torch.equal(got, want)
    for got, want in zip((yb, gb, dxb), single["b"]):
        assert torch.equal(got, want)
    # overwrite mode, no dx: the critic-loss form of the backward pass
    ga2, gb2 = torch.empty_like(ga), torch.empty_like(gb)
    pair.backward(dya, dyb, slot=1, grad_a=ga2, grad_b=gb2)
    ga1 = torch.empty_like(ga)
    a.forward(x, slot=1, train=True)
    a.backward(dya, slot=1, grad=ga1)
    torch.cuda.synchronize()
    assert torch.equal(ga2, ga1) and not torch.equal(ga2, gb2)


def test_pair_pass_issues_the_launches_of_one_single_pass():
    from gops_b200 import _lib
    L = _lib.lib()
    (a, b), _, pair = _net_pair([7, 256, 256, 256, 2], 8192, 13)
    B = 8192
    x = torch.randn(B, 7, device="cuda")
    dy = torch.randn(B, 2, device="cuda")
    ga, gb = torch.empty(a.nparam, device="cuda"), torch.empty(b.nparam, device="cuda")

    def launches(fn):
        c0 = L.gops_b200_launch_count()
        fn()
        return L.gops_b200_launch_count() - c0
    single_f = launches(lambda: a.forward(x, slot=0, train=True))
    pair_f = launches(lambda: pair.forward(x, slot=0, train=True))
    single_b = launches(lambda: a.backward(dy, slot=0, grad=ga, want_dx=True))
    pair_b = launches(lambda: pair.backward(dy, dy, slot=0, grad_a=ga, grad_b=gb, want_dx=True))
    torch.cuda.synchronize()
    assert single_f == pair_f == 4, (single_f, pair_f)
    assert single_b == pair_b == 4 * 4 + 4, (single_b, pair_b)


def test_mismatched_pair_is_refused():
    from gops_b200.ops.layerwise_mlp import LayerwiseMlp, LayerwiseMlpPair
    x = torch.randn(64, 7, device="cuda")
    ref = LayerwiseMlp([7, 64, 64, 2], "gelu", max_batch=256)
    ref.pack(torch.zeros(ref.nparam, device="cuda"))
    for other in (LayerwiseMlp([7, 64, 64, 64, 2], "gelu", max_batch=256), LayerwiseMlp([7, 64, 32, 2], "gelu", max_batch=256),
                  LayerwiseMlp([7, 64, 64, 2], "relu", max_batch=256), LayerwiseMlp([7, 64, 64, 2], "gelu", max_batch=512),
                  LayerwiseMlp([7, 64, 64, 2], "gelu", max_batch=256, slots=2)):
        other.pack(torch.zeros(other.nparam, device="cuda"))
        with pytest.raises(RuntimeError, match="differ in layer sizes"):
            LayerwiseMlpPair(ref, other).forward(x)
    with pytest.raises(RuntimeError, match="distinct"):
        LayerwiseMlpPair(ref, ref).forward(x)
    unpacked = LayerwiseMlp([7, 64, 64, 2], "gelu", max_batch=256)
    with pytest.raises(RuntimeError, match="before mlpnet_pack"):
        LayerwiseMlpPair(ref, unpacked).forward(x)
