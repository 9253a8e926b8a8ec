"""SAC on paired layer-wise wgmma passes (algorithm/sac.py, csrc/sac.cu, apprfunc ActionValue) against the unmodified
reference:
(a) tests/golden/sac_idp*.npz -- consecutive `local_update`s replaying the Gaussian noise the reference drew
    (oracle/make_golden_sac.py), each resumed from the reference's weights: scalars, gradients of q1 / q2 / policy /
    log_alpha, the Adam steps, Polyak targets and the temperature, with and without auto_alpha;
(b) the shipped trained policy (results/SAC/idpendulum, placed in oracle/_ref by build(); its known answers in
    tests/golden/ckpt_sac_idp.npz): state_dict round trip, the closed loop of the mode action through the fused env
    model, q1 / q2 along it, one update from the trained weights;
(c) the reference's own update (oracle/sac_ref.py) at the shipped size: [256,256,256] relu, minibatch 8192 from the
    on-device replay buffer, same batch and noise;
(d) the reference's harness: its registry, factory and ReplayBuffer, next to the unmodified SAC;
(e) the plugin surface: remote update == local update, updates without injected noise.
Bars: scalars 1e-4 relative, gradients 2e-4 relative L2 (BF16x3 six-term forward, three-term gradient products),
log_alpha gradient 2e-5 and value 2e-6, weights by DSAC-T's Adam-step rule."""
import numpy as np
import pytest
import torch

from golden_util import load, rel_l2
from oracle import ref_shim, sac_ref
from test_gpu_dsac import _kwargs as dsac_kwargs
from test_gpu_dsact import _check_weights, _kwargs as dsact_kwargs

pytestmark = pytest.mark.gpu
needs_reference = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not reachable")

TAGS = ("Loss/Critic loss-RL iter", "Loss/Actor loss-RL iter", "SAC/critic_avg_q1-RL iter", "SAC/critic_avg_q2-RL iter",
        "SAC/entropy-RL iter", "SAC/alpha-RL iter")


def _create(kw):
    from gops_b200.create_pkg.create_alg import create_alg
    return create_alg(**dict(kw, use_gpu=True))


def _lr_of(kw):
    return lambda k: kw["policy_learning_rate"] if k.startswith("policy") else kw["q_learning_rate"]


def _grads(net):
    return [p.grad.detach().cpu().numpy() for p in net.parameters()]


def _load(alg, sd):
    alg.load_state_dict({k: torch.as_tensor(np.asarray(v)) for k, v in sd.items()})


def _check_update(alg, tb, want_tb, want_grads, want_sd, kw, tag, tb_rtol=1e-4):
    """tb values, gradients, log_alpha and the post-update weights of one update against the reference's."""
    assert set(TAGS) <= set(tb) and "Time/Algorithm time [ms]-RL iter" in tb
    for k in TAGS:
        ref, got = float(want_tb[k]), tb[k]
        assert abs(got - ref) <= tb_rtol * max(1.0, abs(ref)), (tag, k, got, ref)
    nets = alg.networks
    for net in ("q1", "q2", "policy"):
        names = [f"{net}.{n}" for n, _ in getattr(nets, net).named_parameters()]
        err = rel_l2(_grads(getattr(nets, net)), [want_grads[k] for k in names])
        assert err < 2e-4, (tag, net, err)
    sd = alg.state_dict()
    if kw["auto_alpha"]:
        assert abs(nets.alpha_optimizer.grad - float(want_grads["log_alpha"])) < 2e-5, tag
    assert abs(float(sd["log_alpha"]) - float(want_sd["log_alpha"])) < 2e-6, tag
    _check_weights(sd, want_sd, _lr_of(kw), tag)


# ------------------------------------------------------------------------------------------------ (a) golden updates
@pytest.mark.parametrize("name", sorted(sac_ref.GOLDEN_CASES))
def test_sac_updates_follow_the_reference(name):
    n_iter, _, over = sac_ref.GOLDEN_CASES[name]
    kw = sac_ref.kwargs(**over)
    rec = sac_ref.expand_golden(load(name), kw)
    alg = _create(kw)
    _load(alg, {k[5:]: v for k, v in rec.items() if k.startswith("init/")})
    data = {k[3:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("in_")}
    before = {k: v.clone() for k, v in data.items()}
    log_alpha0 = float(rec["init/log_alpha"])
    for it in range(n_iter):
        if it > 0:        # continue from the reference's own weights so that errors do not compound
            _load(alg, {k.split("/post/")[1]: v for k, v in rec.items() if k.startswith(f"it{it - 1}/post/")})
        alg.noise_override = {k: torch.from_numpy(rec[f"it{it}/{k}"]) for k in ("eps_new", "eps_next")}
        tb = alg.local_update(data, it)
        want_tb = {k.split("/tb/")[1]: v for k, v in rec.items() if k.startswith(f"it{it}/tb/")}
        want_g = {k.split("/grad/")[1]: v for k, v in rec.items() if k.startswith(f"it{it}/grad/")}
        want_sd = {k.split("/post/")[1]: v for k, v in rec.items() if k.startswith(f"it{it}/post/")}
        _check_update(alg, tb, want_tb, want_g, want_sd, kw, (name, it))
        if not kw["auto_alpha"]:
            assert float(alg.state_dict()["log_alpha"]) == log_alpha0 and tb["SAC/alpha-RL iter"] == kw["alpha"]
    assert all(torch.equal(data[k], before[k]) for k in data)           # the batch is not written to


# ------------------------------------------------------------------------------------------------ (b) shipped checkpoint
@needs_reference
def test_shipped_checkpoint_known_answer():
    from gops_b200.create_pkg.create_env_model import create_env_model
    rec = load("ckpt_sac_idp")
    assert sac_ref.checkpoint_sha256() == str(rec["ckpt_sha256"])
    c = sac_ref.CKPT
    kw = sac_ref.kwargs(c["hidden"], c["act"])
    sd0 = {k: v.numpy() for k, v in torch.load(sac_ref.checkpoint_path(), map_location="cpu").items()}
    alg = _create(kw)
    assert set(alg.state_dict()) == set(sd0)
    _load(alg, sd0)
    sd = alg.state_dict()
    for k, v in sd0.items():
        assert np.array_equal(sd[k].cpu().numpy(), v), k
    nets = alg.networks
    pol = nets.policy
    hi, lo = pol.act_high_lim.cuda(), pol.act_low_lim.cuda()
    env = create_env_model("pyth_idpendulum")
    o, d, info, acts = torch.from_numpy(rec["closed_loop_states"][:1]).cuda(), torch.zeros(1).cuda(), {}, []
    for _ in range(5):
        mean = pol(o)[..., :1]
        a = (hi - lo) / 2 * torch.tanh(mean) + (hi + lo) / 2
        acts.append(a.cpu().numpy()[0])
        o, r, d, info = env.forward(o, a, d, info)
    np.testing.assert_allclose(np.stack(acts), rec["closed_loop_actions"], rtol=1e-4, atol=5e-6)
    s, a = torch.from_numpy(rec["closed_loop_states"]).cuda(), torch.from_numpy(rec["closed_loop_actions"]).cuda()
    for q, want in ((nets.q1, rec["closed_loop_q1"]), (nets.q2, rec["closed_loop_q2"])):
        got = q(s, a).cpu().numpy()
        assert got.shape == want.shape
        np.testing.assert_allclose(got, want, rtol=1e-4)
    # one update from the trained weights, against the reference's own on the same batch and noise (whose tb values are
    # the recorded ones: tests/test_oracle_sac.py pins its gradients too)
    data = {k[3:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("in_")}
    noise = {k: torch.from_numpy(rec[f"it0/{k}"]) for k in ("eps_new", "eps_next")}
    want_tb, want_g, want_sd = sac_ref.update(sac_ref.create(kw, sd0), data, noise["eps_new"], noise["eps_next"], 0)
    assert want_tb == {k.split("/tb/")[1]: float(v) for k, v in rec.items() if k.startswith("it0/tb/")}
    alg.noise_override = noise
    tb = alg.local_update(data, 0)
    _check_update(alg, tb, want_tb, want_g, want_sd, kw, "ckpt")


# ------------------------------------------------------------------------------------------------ (c) shipped size
@needs_reference
def test_shipped_size_against_the_reference():
    from gops_b200.trainer.device_buffer import DeviceReplayBuffer
    c = sac_ref.CKPT
    kw = sac_ref.kwargs(c["hidden"], c["act"])
    torch.manual_seed(5)
    alg = _create(kw)
    init = {k: v.detach().cpu().numpy().copy() for k, v in alg.state_dict().items()}
    ref = sac_ref.create(kw, init)
    B, n = 8192, 1 << 15
    buf = DeviceReplayBuffer(6, 1, 1 << 16, device="cuda", seed=3)
    g = torch.Generator().manual_seed(9)
    obs = (torch.rand(n, 6, generator=g) * 2 - 1) * torch.tensor([5, 0.1, 0.1, 0.3, 0.3, 0.3])
    buf.add_batch({"obs": obs, "act": torch.rand(n, 1, generator=g) * 2 - 1, "rew": torch.randn(n, generator=g) * 3,
                   "obs2": obs + 0.05 * torch.randn(n, 6, generator=g), "done": (torch.rand(n, generator=g) < 0.05).float()})
    batch = buf.sample_batch(B)
    assert all(v.is_cuda and v.shape[0] == B for v in batch.values())
    eps_new, eps_next = torch.randn(B, 1, generator=g), torch.randn(B, 1, generator=g)
    want_tb, want_g, want_sd = sac_ref.update(ref, {k: v.cpu() for k, v in batch.items()}, eps_new, eps_next, 0)
    alg.noise_override = {"eps_new": eps_new, "eps_next": eps_next}
    tb = alg.local_update(batch, 0)
    _check_update(alg, tb, want_tb, want_g, want_sd, kw, "B=8192")


# ------------------------------------------------------------------------------------------------ (d) reference harness
@needs_reference
def test_register_binding_and_three_trainer_steps():
    ref_shim.install()
    from gops.create_pkg import create_alg as ref_ca
    from gops.trainer.buffer.replay_buffer import ReplayBuffer
    from gops_b200.algorithm import sac as b200_sac

    kw = sac_ref.kwargs()
    torch.manual_seed(12)
    ref_alg = ref_ca.create_alg(**kw)                                  # the unmodified reference SAC (CPU)
    saved = ref_ca.registry["SAC"]
    try:
        ref_ca.register("SAC", b200_sac.SAC, b200_sac.ApproxContainer)    # INTEGRATION.md section 1
        alg = ref_ca.create_alg(**dict(kw, use_gpu=True))              # reference factory -> fused algorithm
    finally:
        ref_ca.registry["SAC"] = saved
    assert type(alg).__module__ == "gops_b200.algorithm.sac" and ref_ca.registry["SAC"] is saved
    alg.load_state_dict(ref_alg.state_dict())                          # identical start (reference checkpoint keys)
    buf = ReplayBuffer(trainer="off_serial_trainer", seed=0, obsv_dim=6, action_dim=1, buffer_max_size=4096,
                       additional_info={})
    g = torch.Generator().manual_seed(3)
    h = torch.tensor([5, 0.1, 0.1, 0.3, 0.3, 0.3])
    obs = ((torch.rand(2048, 6, generator=g) * 2 - 1) * h).numpy()
    act = (torch.rand(2048, 1, generator=g) * 2 - 1).numpy()
    rew = (torch.randn(2048, generator=g) + 5).numpy()
    buf.add_batch([(o, a, float(r), bool(i % 97 == 0), {}, o + 0.01, {}, 0.0) for i, (o, a, r) in enumerate(zip(obs, act, rew))])
    for it in range(3):
        replay = buf.sample_batch(256)
        eps_new, eps_next = torch.randn(256, 1, generator=g), torch.randn(256, 1, generator=g)
        ref_tb, _, _ = sac_ref.update(ref_alg, replay, eps_new, eps_next, it)
        alg.noise_override = {"eps_new": eps_new, "eps_next": eps_next}
        tb = alg.local_update({k: v.cuda() for k, v in replay.items()}, it)      # off_serial_trainer.py:92-94
        for k in TAGS:
            assert abs(tb[k] - ref_tb[k]) <= (1e-4 if it == 0 else 5e-4) * max(1.0, abs(ref_tb[k])), (it, k)
    ref_alg.load_state_dict({k: v.cpu() for k, v in alg.state_dict().items()})  # the fused checkpoint loads back


# ------------------------------------------------------------------------------------------------ (e) plugin surface
# the soft actor-critic family shares its plugin surface: algorithm -> (kwargs, noise keys, critic gradient keys,
# adjustable parameters)
REMOTE = {
    "SAC": (sac_ref.kwargs, ("eps_new", "eps_next"), ["q1_grad", "q2_grad"],
            ("gamma", "tau", "auto_alpha", "alpha", "target_entropy")),
    "DSAC": (lambda **over: dict(dsac_kwargs((64, 64, 64)), **over), ("eps_new", "eps_next", "z_next"), ["q_grad"],
             ("gamma", "tau", "auto_alpha", "alpha", "bound", "delay_update")),
    "DSACT": (lambda **over: dict(dsact_kwargs((64, 64, 64)), **over), ("eps_new", "eps_next", "z1_next", "z2_next"),
              ["q1_grad", "q2_grad"], ("gamma", "tau", "auto_alpha", "alpha", "delay_update")),
}


def _remote_update_equals_local_update(name):
    make_kw, noise_keys, grad_keys, adjustable = REMOTE[name]
    kw = make_kw()
    torch.manual_seed(7)
    a = _create(kw)
    b = _create(kw)
    b.load_state_dict(a.state_dict())
    B = 300
    g = torch.Generator().manual_seed(8)
    obs = torch.randn(B, 6, generator=g) * 0.3
    data = {"obs": obs.cuda(), "act": (torch.rand(B, 1, generator=g) * 2 - 1).cuda(), "rew": torch.randn(B, generator=g).cuda(),
            "obs2": (obs + 0.05 * torch.randn(B, 6, generator=g)).cuda(), "done": torch.zeros(B).cuda()}
    tbs = []
    for it in range(2):           # DSAC / DSAC-T (delay_update = 2): with and without the policy's step
        noise = {k: torch.randn(B, 1, generator=g) if k.startswith("eps") else torch.randn(B, generator=g)
                 for k in noise_keys}
        a.noise_override = b.noise_override = noise
        tb_a = a.local_update(data, it)
        tb_b, info = b.get_remote_update_info(data, it)
        assert sorted(info) == sorted(["iteration", "log_alpha_grad", "policy_grad"] + grad_keys)
        b.remote_update(info)
        tbs.append((tb_a, tb_b))
        assert set(tb_a) == set(tb_b) and all(tb_a[k] == tb_b[k] for k in tb_a if k != "Time/Algorithm time [ms]-RL iter")
    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    c = _create(make_kw(auto_alpha=False))
    _, info = c.get_remote_update_info(data, 0)
    assert "log_alpha_grad" not in info
    assert c.adjustable_parameters == adjustable
    assert c.target_entropy == -1
    return tbs


def test_remote_update_equals_local_update():
    for tb_a, tb_b in _remote_update_equals_local_update("SAC"):
        assert all(tb_a[k] == tb_b[k] for k in TAGS)


@pytest.mark.parametrize("name", ["DSAC", "DSACT"])
def test_remote_update_equals_local_update_distributional(name):
    _remote_update_equals_local_update(name)


def test_sac_runs_without_injected_noise():
    torch.manual_seed(2)
    alg = _create(sac_ref.kwargs())
    B = 1000
    g = torch.Generator().manual_seed(4)
    obs = torch.randn(B, 6, generator=g) * 0.3
    data = {"obs": obs.cuda(), "act": (torch.rand(B, 1, generator=g) * 2 - 1).cuda(), "rew": torch.randn(B, generator=g).cuda(),
            "obs2": (obs + 0.05 * torch.randn(B, 6, generator=g)).cuda(), "done": torch.zeros(B).cuda()}
    for it in range(3):
        tb = alg.local_update(data, it)
        assert all(np.isfinite(tb[k]) for k in TAGS), tb
    assert all(torch.isfinite(v).all() for v in alg.state_dict().values())

