"""CPU: the oracle's pyth_mobilerobot model (oracle/robot_oracle.py) against the unmodified reference model with the same
obstacle draws: the wrapped envmodel.forward over several steps (crashes, out-of-bounds dones, clipped observations,
frozen done samples included), its autograd gradient, and the SPIL passes on one constraint."""
import os

import numpy as np
import pytest
import torch

from oracle import ref_shim
from oracle import robot_oracle as ro
from oracle import spil_oracle as so

live_reference = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not available")


def inputs(B=512, seed=0):
    """Reset-law states plus crafted rows: obstacle on the robot (crash), robot past x = -2 and |y| = 4 (out of bounds),
    theta beyond 2 pi (clipped), and a quarter of the batch already done."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.tensor([0, -1, -0.6, 0, 0, 0, 0, 0, 3.5, -3, np.pi / 2 - 0.3, 0, 0], dtype=torch.float32)
    hi = torch.tensor([2.7, 1, 0.6, 0.3, 0, 0, 0, 0, 6, 3, np.pi / 2 + 0.3, 0.5, 0], dtype=torch.float32)
    o = lo + torch.rand(B, 13, generator=g) * (hi - lo)
    o[:8, 8:10] = o[:8, 0:2] + 0.3                  # crash
    o[8:16, 0] = -1.98; o[8:16, 3] = -0.3          # about to leave x >= -2
    o[16:24, 1] = 3.95; o[16:24, 2] = 1.5          # about to leave |y| <= 4
    o[24:32, 2] = 6.27; o[24:32, 4] = 1.5          # theta runs past 2 pi: ClipObservation
    o[:, 5], o[:, 6], o[:, 7] = o[:, 1], o[:, 2], o[:, 3] - 0.3
    done = torch.zeros(B)
    done[torch.randperm(B, generator=g)[:B // 4]] = 1.0
    act = torch.rand(B, 2, generator=g) * 2.2 - 1.1
    return o, done, act


def reference_env():
    ref_shim.install()
    from gops.create_pkg.create_env_model import create_env_model
    return create_env_model("pyth_mobilerobot")


@live_reference
def test_forward_matches_the_reference_with_replayed_noise():
    ref = reference_env()
    o, done, _ = inputs()
    B, H = o.shape[0], 6
    noise = ro.draw((H, B), seed=1)
    env = ro.create_env_model([torch.from_numpy(n) for n in noise])
    g = torch.Generator().manual_seed(2)
    ro_, rd_ = o.clone(), done.clone()
    oo, od = o.clone(), done.clone()
    for k in range(H):
        a = torch.rand(B, 2, generator=g) * 2.2 - 1.1
        with ro.replay_normal(noise[k:k + 1]):
            ro_, rr, rd_, rinfo = ref.forward(ro_, a, rd_, {})
        oo, orr, od, oinfo = env.forward(oo, a, od, {})
        assert torch.equal(od, rd_), k
        assert torch.allclose(oo, ro_, rtol=1e-6, atol=1e-6), (k, (oo - ro_).abs().max())
        assert torch.allclose(orr, rr, rtol=1e-6, atol=1e-6), k
        assert torch.allclose(oinfo["constraint"], rinfo["constraint"], rtol=1e-6, atol=1e-6), k
    assert bool(rd_.any()) and not bool(rd_.all())


@live_reference
def test_gradient_matches_the_reference():
    ref = reference_env()
    o, done, a = inputs(256, seed=3)
    noise = ro.draw((1, 256), seed=4)
    grads = []
    for which in ("ref", "oracle"):
        x, u = o.clone().requires_grad_(True), a.clone().requires_grad_(True)
        if which == "ref":
            with ro.replay_normal(noise):
                n, r, d, info = ref.forward(x, u, done, {})
        else:
            n, r, d, info = ro.create_env_model([torch.from_numpy(noise[0])]).forward(x, u, done, {})
        (n.sum() + r.sum() + 3 * info["constraint"].sum()).backward()
        grads.append((x.grad, u.grad))
    for g_ref, g_or in zip(*grads):
        assert torch.allclose(g_ref, g_or, rtol=1e-5, atol=1e-6)


def test_spil_passes_take_one_constraint():
    """spil_oracle's passes on this model: [B, 1] constraints broadcast over its two-column safe record."""
    torch.manual_seed(0)
    o, done, _ = inputs(128, seed=5)
    H = 5
    noise = [torch.from_numpy(n) for n in ro.draw((H, 128), seed=6)]
    from oracle import gops_oracle as orc
    gen = torch.Generator().manual_seed(7)
    mk = lambda sizes: orc.NetSpec(orc.init_mlp(sizes, gen), "relu", "linear",
                                   torch.tensor([0.4, np.pi / 3]), -torch.tensor([0.4, np.pi / 3]))
    pol = mk([13, 64, 64, 2])
    v = orc.NetSpec(orc.init_mlp([13, 64, 64, 1], gen), "relu")
    _, _, issafe = so.spil_loss_value(v, pol, v, ro.create_env_model(noise), {"obs": o, "done": done}, H, 0.99)
    assert torch.equal(issafe[:, 0], issafe[:, 1])
    loss = so.spil_loss_policy(pol, ro.create_env_model(noise), {"obs": o, "done": done}, H, 0.99, 0.5, [0.5])
    assert torch.isfinite(loss)


# ---- the oracle against the reference's recorded SPIL runs (oracle/make_golden_spil_robot.py) --------------------------
def _update_against(rec, prefix, wprefix, data, ctl):
    """One recorded SPIL update: both passes of the oracle on the recorded noise, held to the reference's tb values,
    gradients and controller state.  Returns nothing; asserts."""
    from golden_util import net_from, rel_l2
    noise = rec[prefix + "noise"]
    env = lambda p: ro.create_env_model([torch.from_numpy(n) for n in noise[p]])
    v = net_from(rec, wprefix, "v", "relu", requires_grad=True)
    vt = net_from(rec, wprefix, "v_target", "relu")
    pol = net_from(rec, wprefix, "policy", "relu", requires_grad=True)
    loss_v, vmean, issafe = so.spil_loss_value(v, pol, vt, env(0), data, 25, 0.99)
    loss_v.backward()
    tb = lambda n: float(rec[f"{prefix}tb/{n}-RL iter"])
    assert abs(loss_v.item() - tb("Loss/Critic loss")) <= 2e-6 * max(1.0, abs(tb("Loss/Critic loss")))
    assert abs(vmean.item() - tb("Train/Critic avg value")) <= 2e-6 * max(1.0, abs(vmean.item()))
    keys = [f"{prefix}grad/v.v.{2 * j}.{w}" for j in range(3) for w in ("weight", "bias")]
    assert rel_l2([t.grad.numpy() for pair in v.layers for t in pair], [rec[k] for k in keys]) < 1e-5
    sp = so.safe_probability(issafe)[:1]
    assert np.array_equal(sp, rec[prefix + "safe_prob"]), (sp, rec[prefix + "safe_prob"])
    w_r, w_c = so.spil_weights(ctl, sp)
    assert np.array_equal(ctl["lam"], rec[prefix + "lam"]) and np.array_equal(ctl["delta_i"], rec[prefix + "delta_i"])
    for p in pol.params():
        p.grad = None
    loss_pi = so.spil_loss_policy(pol, env(1), data, 25, 0.99, w_r, w_c)
    loss_pi.backward()
    assert abs(loss_pi.item() - tb("Loss/Actor loss")) <= 2e-6 * max(1.0, abs(tb("Loss/Actor loss")))
    keys = [f"{prefix}grad/policy.pi.{2 * j}.{w}" for j in range(3) for w in ("weight", "bias")]
    assert rel_l2([t.grad.numpy() for pair in pol.layers for t in pair], [rec[k] for k in keys]) < 1e-5


def test_oracle_follows_the_reference_over_four_updates():
    from golden_util import load
    torch.set_num_threads(4)
    rec = load("spil_robot")
    data = {"obs": torch.from_numpy(rec["in_obs"]), "done": torch.from_numpy(rec["in_done"])}
    ctl = so.new_controller(1)
    for it in range(4):
        _update_against(rec, f"it{it}/", "init/" if it == 0 else f"it{it - 1}/post/", data, ctl)


def test_oracle_reproduces_the_shipped_checkpoint():
    """The trained policy's closed loop through the model, and one update from the trained weights."""
    import hashlib
    from golden_util import load, net_from
    rec = load("ckpt_spil_robot")
    path = os.path.join(ref_shim.REFERENCE_ROOT, "results", "SPIL", "mobilerobot", "apprfunc", "apprfunc_16500_opt.pkl")
    if os.path.exists(path):
        with open(path, "rb") as f:
            assert hashlib.sha256(f.read()).hexdigest() == str(rec["sha256"])
    pol = net_from(rec, "ckpt/", "policy", "relu")
    noise = rec["loop/noise"]
    env = ro.create_env_model([torch.from_numpy(n) for n in noise])
    obs, done = torch.from_numpy(rec["loop/obs0"]), torch.zeros(noise.shape[1])
    with torch.no_grad():
        for k in range(noise.shape[0]):
            act = pol.act(obs)
            obs, rew, d, info = env.forward(obs, act, done, {})
            done = d.float()
            for name, got in (("act", act), ("obs", obs), ("rew", rew), ("con", info["constraint"])):
                np.testing.assert_allclose(got.numpy(), rec[f"loop/{name}"][k], rtol=1e-5, atol=1e-5, err_msg=f"{name} {k}")
            assert np.array_equal(done.numpy(), rec["loop/done"][k]), k
    data = {"obs": torch.from_numpy(rec["upd/in_obs"]), "done": torch.from_numpy(rec["upd/in_done"])}
    _update_against(rec, "upd/", "ckpt/", data, so.new_controller(1))
