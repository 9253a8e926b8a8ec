"""SPIL on pyth_mobilerobot (fused mma.sync rollout, constraint mode 4 with the model's one constraint of the raw next
state, obstacle noise read from a device buffer): four updates of the unmodified reference's SPIL and the known answers
of its shipped checkpoint (tests/golden/spil_robot.npz, ckpt_spil_robot.npz; oracle/make_golden_spil_robot.py), both on
the reference's recorded noise; envmodel.forward against the unmodified reference with replayed noise, both passes against the fp64 oracle at B = 1024 and at a ragged B of about 2^16 with done samples, the
one-constraint controller against its NumPy statement, the launch count, a bit-identical repeat, the refusals and the
example script."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import load, rel_l2
from oracle import gops_oracle as orc
from oracle import ref_shim
from oracle import robot_oracle as ro
from oracle import spil_oracle as so

pytestmark = pytest.mark.gpu

H = 25
LAUNCHES_PER_UPDATE = 13   # as on pyth_veh3dofconti_errcstr: the noise draws are torch launches, not the library's
ACT_HI = np.array([0.4, np.pi / 3], np.float32)


def _kwargs(**over):
    kw = dict(env_id="pyth_mobilerobot", algorithm="SPIL", seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=13, action_dim=2, action_high_limit=ACT_HI, action_low_limit=-ACT_HI,
              policy_func_name="DetermPolicy", policy_func_type="MLP", policy_hidden_sizes=[64, 64],
              policy_hidden_activation="relu", policy_act_distribution="default", policy_learning_rate=3e-4,
              value_func_name="StateValue", value_func_type="MLP", value_hidden_sizes=[64, 64],
              value_hidden_activation="relu", value_learning_rate=2e-3, forward_step=H, constraint_dim=1,
              gamma=0.99, tau=0.005)
    kw.update(over)
    return kw


def _alg(**kw):
    from gops_b200.create_pkg.create_alg import create_alg
    return create_alg(**_kwargs(**kw))


def _batch(B, seed, done_frac=0.2):
    """Reset-law states; some obstacles moved onto the robot (crashes within the horizon) and some samples done."""
    from gops_b200.trainer.device_sampler import sample_mobilerobot
    d = sample_mobilerobot(B, "cuda", seed=seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    near = torch.rand(B, generator=g, device="cuda") < 0.1
    d["obs"][near, 8] = d["obs"][near, 0] + 0.9
    d["obs"][near, 9] = d["obs"][near, 1]
    d["obs"][near, 10] = float(np.float32(np.pi))
    d["obs"][near, 11] = 0.4
    d["done"] = (torch.rand(B, generator=g, device="cuda") < done_frac).float()
    return d


def _net(alg, name, dtype):
    seq = getattr(alg.networks, name)
    mods = [m for m in seq.modules() if isinstance(m, torch.nn.Linear)]
    layers = [(m.weight.detach().cpu().to(dtype).clone().requires_grad_(True),
               m.bias.detach().cpu().to(dtype).clone().requires_grad_(True)) for m in mods]
    if name == "policy":
        return orc.NetSpec(layers, "relu", "linear", torch.tensor(ACT_HI, dtype=dtype), -torch.tensor(ACT_HI, dtype=dtype))
    return orc.NetSpec(layers, "relu")


def _grad(alg, name):
    return [p.grad.detach().cpu().numpy().astype(np.float64) for p in getattr(alg.networks, name).parameters()]


def _golden_update(alg, rec, prefix, data, it):
    """One local_update on the reference's recorded noise, held to its tb values (1e-4), gradients (1e-3 rel. L2) and
    controller state (equal)."""
    noise = torch.from_numpy(rec[prefix + "noise"]).cuda()
    alg.noise_override = {"value": noise[0], "policy": noise[1]}
    tb = alg.local_update(data, it)
    for tag in ("Loss/Critic loss-RL iter", "Train/Critic avg value-RL iter", "Loss/Actor loss-RL iter"):
        ref = float(rec[f"{prefix}tb/{tag}"])
        assert abs(tb[tag] - ref) <= 1e-4 * max(1.0, abs(ref)), (prefix, tag, tb[tag], ref)
    for net in ("v", "policy"):
        got = {n: p.grad.detach().cpu().numpy() for n, p in getattr(alg.networks, net).named_parameters()}
        keys = sorted(got)
        err = rel_l2([got[k] for k in keys], [rec[f"{prefix}grad/{net}.{k}"] for k in keys])
        assert err < 1e-3, (prefix, net, err)
    assert np.array_equal(alg.safe_prob, rec[prefix + "safe_prob"]), (prefix, alg.safe_prob, rec[prefix + "safe_prob"])
    np.testing.assert_array_equal(alg.lam, rec[prefix + "lam"])
    np.testing.assert_array_equal(alg.delta_i, rec[prefix + "delta_i"])


def _load(alg, rec, prefix):
    alg.load_state_dict({k[len(prefix):]: torch.from_numpy(v) for k, v in rec.items() if k.startswith(prefix)})


def test_four_updates_follow_the_reference():
    rec = load("spil_robot")
    alg = _alg()
    data = {"obs": torch.from_numpy(rec["in_obs"]).cuda(), "done": torch.from_numpy(rec["in_done"]).cuda()}
    for it in range(4):      # each from the reference's weights; the controller state carries on on the device
        _load(alg, rec, "init/" if it == 0 else f"it{it - 1}/post/")
        _golden_update(alg, rec, f"it{it}/", data, it)


def test_shipped_checkpoint_known_answers():
    """results/SPIL/mobilerobot's trained policy: its closed loop through the model on the recorded noise, and one SPIL
    update from the trained weights."""
    from gops_b200.create_pkg.create_env_model import create_env_model
    rec = load("ckpt_spil_robot")
    alg = _alg()
    _load(alg, rec, "ckpt/")
    env = create_env_model("pyth_mobilerobot")
    noise = rec["loop/noise"]
    obs = torch.from_numpy(rec["loop/obs0"]).cuda()
    done = torch.zeros(obs.shape[0], device="cuda")
    with torch.no_grad():
        for k in range(noise.shape[0]):
            act = alg.networks.policy(obs)
            env.unwrapped.noise_override = torch.from_numpy(noise[k])
            obs, rew, d, info = env.forward(obs, act, done, {})
            done = d.float()
            for name, got in (("act", act), ("obs", obs), ("rew", rew), ("con", info["constraint"])):
                np.testing.assert_allclose(got.cpu().numpy(), rec[f"loop/{name}"][k], rtol=1e-4, atol=1e-4,
                                           err_msg=f"{name} step {k}")
            assert np.array_equal(done.cpu().numpy(), rec["loop/done"][k]), k
    data = {"obs": torch.from_numpy(rec["upd/in_obs"]).cuda(), "done": torch.from_numpy(rec["upd/in_done"]).cuda()}
    _golden_update(alg, rec, "upd/", data, 0)


def test_forward_matches_the_reference_with_replayed_noise():
    from gops_b200.create_pkg.create_env_model import create_env_model
    ref_shim.install()
    from gops.create_pkg.create_env_model import create_env_model as ref_create
    ref, env = ref_create("pyth_mobilerobot"), create_env_model("pyth_mobilerobot")
    B, steps = 4096, 8
    d = _batch(B, seed=11, done_frac=0.25)
    d["obs"][:64, 2] = 6.2                          # theta runs past 2 pi: ClipObservation
    d["obs"][:64, 4] = 1.5
    noise = ro.draw((steps, B), seed=12)
    o_g, d_g = d["obs"].clone(), d["done"].clone()
    o_r, d_r = d["obs"].cpu(), d["done"].cpu()
    g = torch.Generator().manual_seed(13)
    clipped = 0
    for k in range(steps):
        a = torch.rand(B, 2, generator=g) * 2.2 - 1.1
        env.unwrapped.noise_override = torch.from_numpy(noise[k])
        o_g, r_g, d_g, info = env.forward(o_g, a.cuda(), d_g, {})
        with ro.replay_normal(noise[k:k + 1]):
            o_r, r_r, d_r, rinfo = ref.forward(o_r, a, d_r, {})
        clipped += int((o_r[:, 2].abs() >= np.float32(2 * np.pi)).sum())
        torch.testing.assert_close(o_g.cpu(), o_r, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(r_g.cpu(), r_r, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(info["constraint"].cpu(), rinfo["constraint"], rtol=1e-5, atol=1e-5)
        assert torch.equal(d_g.cpu(), d_r), k
        d_g = d_g.float()
    assert clipped > 0 and 0 < int(d_r.sum()) < B


@pytest.mark.parametrize("B", [1024, (1 << 16) + 37])
def test_passes_match_the_fp64_oracle(B):
    alg = _alg()
    data = _batch(B, seed=B % 1000)
    nv = torch.from_numpy(ro.draw((H, B), seed=1)).cuda()
    npol = torch.from_numpy(ro.draw((H, B), seed=2)).cuda()
    alg.noise_override = {"value": nv, "policy": npol}
    pol, v, vt = (_net(alg, n, torch.float64) for n in ("policy", "v", "v_target"))
    tb = alg.local_update(data, 0)
    w = alg._ctl()[1].cpu().numpy()
    cpu = {k: t.cpu() for k, t in data.items()}
    cpu64 = dict(cpu, obs=cpu["obs"].double())
    env_v = ro.create_env_model([n.double() for n in nv.cpu()], dtype=torch.float64)
    loss_v, vmean, issafe = so.spil_loss_value(v, pol, vt, env_v, cpu64, H, 0.99)
    loss_v.backward()
    assert abs(tb["Loss/Critic loss-RL iter"] - loss_v.item()) <= 1e-4 * max(1.0, abs(loss_v.item()))
    assert abs(tb["Train/Critic avg value-RL iter"] - vmean.item()) <= 1e-4 * max(1.0, abs(vmean.item()))
    assert rel_l2(_grad(alg, "v"), [t.grad.numpy() for pair in v.layers for t in pair]) < 1e-3
    # safe flags sit on fp32 constraint values: at most a handful of trajectories may flip against fp64
    assert abs(float(alg.safe_prob[0]) - float(issafe[:, 0].mean())) * B <= 3 + 1e-3 * B
    assert alg.safe_prob.shape == (1,) and alg.lam.shape == (1,) and alg.delta_i.shape == (1,)
    env_p = ro.create_env_model([n.double() for n in npol.cpu()], dtype=torch.float64)
    for p in pol.params():
        p.grad = None
    loss_pi = so.spil_loss_policy(pol, env_p, cpu64, H, 0.99, float(w[0]), [float(w[1])])
    loss_pi.backward()
    assert abs(tb["Loss/Actor loss-RL iter"] - loss_pi.item()) <= 1e-4 * max(1.0, abs(loss_pi.item()))
    assert rel_l2(_grad(alg, "policy"), [t.grad.numpy() for pair in pol.layers for t in pair]) < 1e-3


def test_one_constraint_controller_equals_numpy():
    """chance_thre1 = 0 on a zero safe count: lam_1 = 0 exactly, and the weights are the reference's
    1 / (1 + lam.sum()), lam / (1 + lam.sum()) bit for bit, over a sequence of safe probabilities."""
    from gops_b200 import _lib
    B = 1024
    state = torch.zeros(6, dtype=torch.float64, device="cuda")
    w = torch.zeros(3, dtype=torch.float32, device="cuda")
    ctl = so.new_controller(1)
    for count in (1000, 990, 700, 1024, 850, 0, 1010, 1000):
        tail = torch.tensor([0.0, 0.0, float(count), 0.0], device="cuda")
        _lib.check(_lib.lib().gops_b200_spil_controller(_lib.ptr(tail), B, 60.0, 0.02, 0.0, 0.97, 0.0, _lib.ptr(state),
                                                        _lib.ptr(w), _lib.stream_ptr()))
        sp = np.array([np.float32(count) / np.float32(B)], dtype=np.float32)
        w_r, w_c = so.spil_weights(ctl, sp)
        st, wd = state.cpu().numpy(), w.cpu().numpy()
        assert st[1] == 0.0 and st[5] == 0.0 and wd[2] == 0.0
        assert st[4] == ctl["lam"][0] and st[0] == ctl["delta_i"][0], (count, st, ctl)
        assert wd[0] == np.float32(w_r) and wd[1] == np.float32(w_c[0]), (count, wd, w_r, w_c)


def test_launches_and_bit_identical_repeat():
    from gops_b200 import _lib
    data = _batch(2048, seed=21)
    runs = []
    for _ in range(2):
        torch.manual_seed(0)      # same initial weights and the same noise generator seed
        alg = _alg()
        launches = []
        for it in range(3):
            c0 = _lib.lib().gops_b200_launch_count()
            tb = alg.local_update(data, it)
            torch.cuda.synchronize()
            launches.append(_lib.lib().gops_b200_launch_count() - c0)
            assert all(math.isfinite(tb[k]) for k in ("Loss/Critic loss-RL iter", "Loss/Actor loss-RL iter"))
        assert launches == [LAUNCHES_PER_UPDATE] * 3, launches
        runs.append(({k: v.detach().cpu().clone() for k, v in alg.state_dict().items()}, alg.lam.copy()))
    for k in runs[0][0]:
        assert torch.equal(runs[0][0][k], runs[1][0][k]), k
    assert np.array_equal(runs[0][1], runs[1][1])


def test_refusals():
    from gops_b200 import _lib
    with pytest.raises(ValueError, match="constraint_dim"):
        _alg(constraint_dim=2)
    with pytest.raises(ValueError, match="repeat_num"):
        _alg(repeat_num=2)
    alg = _alg()
    alg.kernel_path = "tc"
    with pytest.raises(RuntimeError, match="wgmma"):
        alg.local_update(_batch(256, seed=3), 0)
    # a rollout without its noise buffer is refused, not run on stale draws
    alg = _alg()
    plan = alg._plan(_lib.ALG_INFADP_VALUE, alg.networks.policy, alg.networks.v, H, 0.99)
    _lib.check(_lib.lib().gops_b200_plan_set_model_io(plan.handle, None, None))
    assert _lib.lib().gops_b200_plan_set_constraint(plan.handle, 4, 1.0) == 0
    nets = alg.networks
    with pytest.raises(RuntimeError, match="noise"):
        alg._rollout_grad(plan, _batch(256, seed=4), nets.v.flat_params, nets.policy.flat_params, nets.v.flat_params,
                          nets.v_target.flat_params)


def test_example_script_trains():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "example_train", "spil_mlp_mobilerobot_b200.py"),
                          "--max_iteration", "21", "--eval_interval", "10", "--log_save_interval", "5"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    losses = [float(x) for line in out.stdout.splitlines() for x in
              [part.split(":")[1].strip(" }") for part in line.split(",") if "loss-RL iter" in part]]
    assert len(losses) >= 8 and all(math.isfinite(x) for x in losses), out.stdout[-2000:]
