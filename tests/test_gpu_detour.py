"""env_gen_ocp veh3dof_tracking_detour (N3: the model of the reference's fhadp_mlp_veh3ddetour example) and its sibling
veh3dof_tracking_surrcstr with FHADP and the
constrained variants FHADPExterior / FHADPLagrangian / FHADPInterior on the layer-wise wgmma path (csrc/lw_detour.cuh):
against the unmodified reference's golden vectors (two consecutive updates) and against the fp64 oracle on a fresh
ragged batch with done samples -- whose state keeps evolving behind the frozen observation and keeps paying the
constraint -- for the 64-wide nets of the goldens and the [256, 256] nets of the reference's example."""
import numpy as np
import pytest
import torch

from golden_util import inputs_from, load, net_from, rel_l2
from oracle import gops_oracle as orc

pytestmark = pytest.mark.gpu

EXTRA = {"FHADP": {}, "FHADPExterior": dict(penalty=2.0, penalty_increase=1.5, penalty_delay=1),
         "FHADPInterior": dict(penalty=2.0, penalty_increase=1.5, penalty_delay=1),
         "FHADPLagrangian": dict(multiplier=1.5, multiplier_lr=5e-2, multiplier_delay=1)}
MODE = {"FHADPExterior": "exterior", "FHADPLagrangian": "lagrangian", "FHADPInterior": "interior"}
GRAD_RTOL = 2e-4


def _alg(algname, hidden=64, P=10, env_id="veh3dof_tracking_detour", **over):
    from gops_b200.create_pkg.create_alg import create_alg
    kw = dict(env_id=env_id, algorithm=algname, seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=6 + 4 * P + 4, action_dim=2, action_high_limit=np.ones(2, np.float32),
              action_low_limit=-np.ones(2, np.float32), policy_func_name="FiniteHorizonPolicy", policy_func_type="MLP",
              policy_hidden_sizes=[hidden, hidden], policy_hidden_activation="elu", policy_act_distribution="default",
              policy_learning_rate=1e-3, value_func_type="MLP", pre_horizon=P, gamma=0.97)
    kw.update(EXTRA[algname])
    kw.update(over)
    return create_alg(**kw)


def _gpu_data(data):
    from gops_b200.env.env_gen_ocp.pyth_base import ContextState, State
    robot, reference, t, surr = data["state"]
    out = dict(data)
    out["state"] = State(robot_state=robot, context_state=ContextState(reference=reference, constraint=surr, t=t))
    return out


def _noise_floor(rec, it, mode, coef, env_id="veh3dof_tracking_detour"):
    """Distance between the reference's own fp32 gradient and the fp64 evaluation of the same formulas: the log barrier
    (and the norm in the collision distance) amplify fp32 round-off for samples near the boundary."""
    env64 = orc.create_env_model(env_id, dtype=torch.float64, pre_horizon=10)
    pol64 = net_from(rec, "init/" if it == 0 else "it0/post/", "policy", "elu", torch.float64, requires_grad=True)
    pol64.time_input = True
    d64 = inputs_from(rec, "veh3dof_tracking_detour", torch.float64)
    if mode is None:
        l64 = orc.fhadp_loss(pol64, env64, d64, 10, 0.97)
    else:
        l64 = orc.fhadp_constrained_loss(mode, pol64, env64, d64, 10, 0.97, coef)[0]
    l64.backward()
    order = [f"it{it}/grad/policy.pi.{2 * j}.{w}" for j in range(3) for w in ("weight", "bias")]
    return rel_l2([t.grad.numpy() for pair in pol64.layers for t in pair], [rec[k] for k in order])


@pytest.mark.parametrize("algname,case", [(a, "detour") for a in sorted(EXTRA)] + [("FHADPExterior", "surrcstr")])
def test_two_updates_follow_the_reference(algname, case):
    rec = load(case + "_" + algname.lower())
    env_id = "veh3dof_tracking_" + case
    alg = _alg(algname, env_id=env_id)
    alg.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("init/")})
    data = _gpu_data(inputs_from(rec, "veh3dof_tracking_detour"))
    for it in (0, 1):
        if it == 1:
            alg.load_state_dict({k.split("/post/")[1]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("it0/post/")})
        tb = alg.local_update(data, it)
        assert alg.last_kernel_path() == "tc"
        for k in (k for k in rec if k.startswith(f"it{it}/tb/")):
            ref = float(rec[k])
            got = tb[k.split("/tb/")[1]]
            assert abs(got - ref) <= 1e-4 * max(1.0, abs(ref)), (it, k, got, ref)
        keys = sorted(k for k in rec if k.startswith(f"it{it}/grad/policy."))
        named = dict(alg.networks.policy.named_parameters())
        err = rel_l2([named[k.split("/grad/policy.")[1]].grad.cpu().numpy() for k in keys], [rec[k] for k in keys])
        coef = None
        if algname in MODE:
            coef = 2.0 * 1.5 ** it if algname != "FHADPLagrangian" else float(rec[f"it{it}/tb/Loss/Lagrange multiplier-RL iter"])
        bar = max(GRAD_RTOL, 3.0 * _noise_floor(rec, it, MODE.get(algname), coef, env_id))
        assert err < bar, (it, err, bar)


@pytest.mark.parametrize("algname,hidden,env_id", [(a, h, "veh3dof_tracking_detour") for a in sorted(EXTRA) for h in (64, 256)]
                         + [("FHADPInterior", 256, "veh3dof_tracking_surrcstr"), ("FHADP", 64, "veh3dof_tracking_surrcstr")])
def test_against_fp64_oracle_with_done_samples(algname, hidden, env_id):
    B, P = 777, 12
    torch.manual_seed(B + hidden)
    alg = _alg(algname, hidden=hidden, P=P, env_id=env_id, reward_scale=0.5, reward_shift=0.3)
    data = orc.sample_inputs(env_id, B, seed=B, pre_horizon=P)
    data["done"][::5] = 1.0
    env = orc.create_env_model(env_id, dtype=torch.float64, pre_horizon=P, reward_scale=0.5, reward_shift=0.3)
    pi = alg.networks.policy.pi
    layers = [(pi[j].weight.detach().cpu().double().requires_grad_(True), pi[j].bias.detach().cpu().double().requires_grad_(True))
              for j in (0, 2, 4)]
    pol = orc.NetSpec(layers, "elu", "linear", torch.ones(2, dtype=torch.float64), -torch.ones(2, dtype=torch.float64),
                      time_input=True)
    d64 = {"obs": data["obs"].double(), "done": data["done"].double(),
           "state": tuple(v.double() if torch.is_tensor(v) else v for v in data["state"])}
    if algname == "FHADP":
        loss = orc.fhadp_loss(pol, env, d64, P, 0.97)
        l_c = feas = None
    else:
        coef = 2.0 if algname != "FHADPLagrangian" else 1.5
        loss, l_r, l_c, feas = orc.fhadp_constrained_loss(MODE[algname], pol, env, d64, P, 0.97, coef)
    loss.backward()
    tb = alg.get_remote_update_info(_gpu_data(data), 0)[0]
    assert alg.last_kernel_path() == "tc"
    assert abs(tb["Loss/Actor loss-RL iter"] - loss.item()) <= 1e-4 * max(1.0, abs(loss.item()))
    if l_c is not None:
        assert abs(tb["Loss/Actor constraint loss-RL iter"] - l_c.item()) <= 1e-4 * max(1.0, abs(l_c.item()))
    if algname == "FHADPInterior":
        assert abs(tb["Loss/Feasible ratio-RL iter"] - float(feas)) < 1e-6
        assert 0.05 < float(feas) < 0.95            # the batch mixes feasible and colliding rollouts
    got = [p.grad.detach().cpu().numpy() for p in alg.networks.policy.parameters()]
    want = [t.grad.numpy() for pair in layers for t in pair]
    # fp32 evaluation of the interior-point barrier against fp64: same conditioning argument as in the golden test
    bar = 5e-3 if algname == "FHADPInterior" else GRAD_RTOL
    assert rel_l2(got, want) < bar


@pytest.mark.parametrize("env_id", ["veh3dof_tracking_detour", "veh3dof_tracking_surrcstr"])
def test_single_step_forward_matches_the_oracle(env_id):
    """envmodel.forward (EnvModel.forward inside the wrapper chain): three consecutive steps incl. samples that arrive done
    -- frozen observation, zero reward, state still advancing -- and info["constraint"] of the incoming state."""
    from gops_b200.create_pkg.create_env_model import create_env_model
    B, P = 300, 10
    env = create_env_model(env_id=env_id, pre_horizon=P, reward_scale=0.5, reward_shift=0.1)
    ref = orc.create_env_model(env_id, pre_horizon=P, reward_scale=0.5, reward_shift=0.1)
    d = orc.sample_inputs(env_id, B, seed=9, pre_horizon=P)
    d["done"][::4] = 1.0
    g = _gpu_data(d)
    obs, done, info = g["obs"].cuda(), g["done"].cuda(), {"state": g["state"]}
    o_ref, d_ref, i_ref = d["obs"], d["done"], d
    gen = torch.Generator().manual_seed(3)
    for _ in range(3):
        act = torch.rand(B, 2, generator=gen) * 2.4 - 1.2            # beyond the action box: exercises scale + clip
        obs, rew, done, info = env.forward(obs, act.cuda(), done, info)
        o_ref, r_ref, d_ref, i_ref = ref.forward(o_ref, act, d_ref, i_ref)
        assert torch.allclose(obs.cpu(), o_ref, rtol=1e-5, atol=2e-5)
        assert torch.allclose(rew.cpu(), r_ref, rtol=1e-5, atol=1e-5)
        assert torch.equal(done.cpu().bool(), d_ref.bool())
        assert torch.allclose(info["state"].robot_state.cpu(), i_ref["state"][0], rtol=1e-5, atol=1e-5)
        assert torch.allclose(info["constraint"].cpu(), i_ref["constraint"], rtol=1e-5, atol=1e-5)
        done = done.float()


def test_device_sampler_feeds_the_interior_point_update():
    """N2 meets N3: batches drawn on the device (static obstacle 20 m ahead, the reference's detour context) through the
    example's configuration -- FHADPInterior, [256, 256] elu, pre_horizon 30 -- a few updates, finite and improving."""
    from gops_b200.trainer.device_trainer import DeviceStateSampler
    torch.manual_seed(0)
    P = 30
    alg = _alg("FHADPInterior", hidden=256, P=P, gamma=1.0, penalty=1.0, penalty_increase=1.1, penalty_delay=100,
               policy_learning_rate=3e-5)
    sampler = DeviceStateSampler("veh3dof_tracking_detour", "cuda", seed=5, pre_horizon=P)
    data = sampler.sample(2048)
    assert data["obs"].shape == (2048, 6 + 4 * P + 4) and data["state"].context_state.constraint.shape == (2048, P + 1, 1, 5)
    losses = []
    for it in range(6):
        tb = alg.local_update(data, it)
        losses.append(tb["Loss/Actor loss-RL iter"])
        assert np.isfinite(losses[-1]) and 0.0 <= tb["Loss/Feasible ratio-RL iter"] <= 1.0
    assert losses[-1] < losses[0]


def test_example_script_trains_and_evaluates():
    """example_train/fhadp_mlp_veh3ddetour_b200.py for a few iterations: device sampler -> interior-point update ->
    batched evaluation through envmodel.forward (the detour model's own single-step kernel)."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "example_train", "fhadp_mlp_veh3ddetour_b200.py"),
                          "--max_iteration", "21", "--eval_interval", "10", "--replay_batch_size", "1024", "--pre_horizon", "12"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "Loss/Feasible ratio-RL iter" in out.stdout and "TAR" in out.stdout, out.stdout[-2000:]
