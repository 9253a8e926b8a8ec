"""SPIL on pyth_veh3dofconti_errcstr (fused rollout kernel, constraint mode 4; device PI controller): against the
unmodified reference's golden vectors (four consecutive updates, safe probability near and far from the threshold),
against the fp64 oracle on a fresh ragged batch with done samples, the controller kernel against its NumPy statement,
the launch count and controller trajectory of an update loop, the refusals, and the example script."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import inputs_from, load, net_from, oracle_chunked, rel_l2
from oracle import gops_oracle as orc
from oracle import spil_oracle as so

pytestmark = pytest.mark.gpu

TOLS = {"spil_near": (3.0, 2.3), "spil_far": (0.9, 1.6)}      # (y_error_tol, u_error_tol) of oracle/make_golden_spil.py
GRAD_RTOL = 1e-3        # pyth_veh3dofconti: fp32 finite-difference heading in the reference (see test_gpu_constrained.py)
LAUNCHES_PER_UPDATE = 13   # value pass 5 (3 packs, rollout, reduction), Adam, controller, policy pass 3, Adam, 2 Polyak
TB = {"loss_critic": "Loss/Critic loss-RL iter", "critic_avg_value": "Train/Critic avg value-RL iter",
      "loss_actor": "Loss/Actor loss-RL iter"}


def _kwargs(y_tol=3.0, u_tol=2.3, **over):
    kw = dict(env_id="pyth_veh3dofconti_errcstr", algorithm="SPIL", seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=46, action_dim=2, action_high_limit=np.ones(2, np.float32),
              action_low_limit=-np.ones(2, np.float32), policy_func_name="DetermPolicy", policy_func_type="MLP",
              policy_hidden_sizes=[64, 64], policy_hidden_activation="relu", policy_act_distribution="default",
              policy_learning_rate=1e-3, value_func_name="StateValue", value_func_type="MLP", value_hidden_sizes=[64, 64],
              value_hidden_activation="relu", value_learning_rate=1e-3, pre_horizon=10, forward_step=10, constraint_dim=2,
              y_error_tol=y_tol, u_error_tol=u_tol, gamma=0.99, tau=0.005)
    kw.update(over)
    return kw


def _alg(*a, **kw):
    from gops_b200.create_pkg.create_alg import create_alg
    return create_alg(**_kwargs(*a, **kw))


def _with_replay_keys(data):
    """The replay batch the reference hands over (act / rew / obs2 / constraint are read only to be overwritten)."""
    B = data["obs"].shape[0]
    return dict(data, act=torch.zeros(B, 2), rew=torch.zeros(B), obs2=data["obs"].clone(), constraint=torch.zeros(B, 2))


def _grads(alg, net):
    return dict((n, p.grad.detach().cpu().numpy()) for n, p in getattr(alg.networks, net).named_parameters())


@pytest.mark.parametrize("name", sorted(TOLS))
def test_four_updates_follow_the_reference(name):
    rec = load(name)
    alg = _alg(*TOLS[name])
    alg.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("init/")})
    data = _with_replay_keys(inputs_from(rec, "pyth_veh3dofconti"))
    for it in range(4):
        if it > 0:      # continue from the reference's weights; the controller state carries on on the device
            alg.load_state_dict({k.split("/post/")[1]: torch.from_numpy(v) for k, v in rec.items()
                                 if k.startswith(f"it{it - 1}/post/")})
        pre = {k: v.detach().cpu().numpy().copy() for k, v in alg.state_dict().items()}
        tb = alg.local_update(data, it)
        for tag in TB.values():
            ref = float(rec[f"it{it}/tb/{tag}"])
            assert abs(tb[tag] - ref) <= 1e-4 * max(1.0, abs(ref)), (it, tag, tb[tag], ref)
        for net in ("v", "policy"):
            got = _grads(alg, net)
            keys = sorted(got)
            err = rel_l2([got[k] for k in keys], [rec[f"it{it}/grad/{net}.{k}"] for k in keys])
            assert err < GRAD_RTOL, (it, net, err)
        assert np.array_equal(alg.safe_prob, rec[f"it{it}/safe_prob"]), (it, alg.safe_prob, rec[f"it{it}/safe_prob"])
        np.testing.assert_array_equal(alg.lam, rec[f"it{it}/lam"])
        np.testing.assert_array_equal(alg.delta_i, rec[f"it{it}/delta_i"])
        # post-update state_dict: the update (Adam step, Polyak average) of every tensor against the reference's.  Adam
        # moves an entry by about lr whatever its gradient, so an entry whose tiny gradient changes sign within the
        # gradient tolerance may move the other way: at most 2 lr per entry, a small share of the step's norm.
        post = {k: v.detach().cpu().numpy() for k, v in alg.state_dict().items()}
        for k, v in post.items():
            ref = rec[f"it{it}/post/{k}"]
            if "act_" in k:
                assert np.array_equal(v, ref), k
                continue
            step_ref = ref.astype(np.float64) - pre[k]
            err = rel_l2([v.astype(np.float64) - pre[k]], [step_ref])
            assert err < 0.1 and np.abs(v.astype(np.float64) - ref).max() <= 2.5e-3, (it, k, err)


def test_against_fp64_oracle_with_done_samples():
    check_against_fp64_oracle(777)


def check_against_fp64_oracle(B, y_tol=2.0, u_tol=2.0):
    """test_against_fp64_oracle_with_done_samples at any batch size (the oracle runs in chunks of 32768 samples).
    Returns the algorithm."""
    torch.manual_seed(B)
    alg = _alg(y_tol, u_tol, reward_scale=0.5)
    data = orc.sample_inputs("pyth_veh3dofconti", B, seed=B, pre_horizon=10)
    data["done"][::5] = 1.0
    env = orc.create_env_model("pyth_veh3dofconti_errcstr", dtype=torch.float64, pre_horizon=10, y_error_tol=y_tol,
                               u_error_tol=u_tol, reward_scale=0.5)
    d64 = {k: (v.double() if v.is_floating_point() else v) for k, v in data.items()}
    sd = {k: v.detach().cpu() for k, v in alg.state_dict().items()}
    sd_np = {k: v.numpy() for k, v in sd.items()}
    v = net_from(sd_np, "", "v", "relu", torch.float64, requires_grad=True)
    vt = net_from(sd_np, "", "v_target", "relu", torch.float64)
    pol = net_from(sd_np, "", "policy", "relu", torch.float64, requires_grad=True)
    tb, _ = alg.get_remote_update_info(_with_replay_keys(data), 0)
    torch.cuda.synchronize()
    # value pass
    def value_chunk(d):
        loss_v, vmean, issafe = so.spil_loss_value(v, pol, vt, env, d, 10, 0.99)
        return (loss_v, vmean, *issafe.mean(0))
    loss_v, g_v, (vmean, *safe) = oracle_chunked(value_chunk, d64, v.params())
    assert abs(tb[TB["loss_critic"]] - loss_v) <= 1e-4 * max(1.0, abs(loss_v))
    assert abs(tb[TB["critic_avg_value"]] - vmean) <= 1e-4 * max(1.0, abs(vmean))
    got = _grads(alg, "v")
    assert rel_l2([got[f"v.{2 * j}.{w}"] for j in range(3) for w in ("weight", "bias")],
                  [g.numpy() for g in g_v]) < GRAD_RTOL
    # safe counts: exact unless a constraint value lies within fp32 round-off of 0
    o, dn, info, near = d64["obs"], d64["done"], d64, torch.zeros(B, 2, dtype=torch.bool)
    with torch.no_grad():
        for _ in range(10):
            o, _, dn, info = env.forward(o, pol.act(o), dn, info)
            near |= info["constraint"].abs() < 1e-4
    counts = np.array(safe) * B
    got_counts = np.rint(alg.safe_prob.astype(np.float64) * B)      # safe_prob is a float32 ratio of counts
    assert np.all(np.abs(got_counts - counts) <= near.sum(0).numpy() + 1e-3), (got_counts, counts)
    # policy pass with the weights the controller left on the device
    w = alg._ctl()[1].cpu().numpy().astype(np.float64)
    loss_pi, g_pi, _ = oracle_chunked(lambda d: so.spil_loss_policy(pol, env, d, 10, 0.99, w[0], w[1:]), d64,
                                      pol.params())
    assert abs(tb[TB["loss_actor"]] - loss_pi) <= 1e-4 * max(1.0, abs(loss_pi))
    got = _grads(alg, "policy")
    assert rel_l2([got[f"pi.{2 * j}.{w}"] for j in range(3) for w in ("weight", "bias")],
                  [g.numpy() for g in g_pi]) < GRAD_RTOL
    return alg


@pytest.mark.parametrize("Kp,Ki,Kd", [(60, 0.02, 0), (60, 0.02, 0.5), (6000, 0.3, 1e4)])
def test_controller_kernel_matches_numpy(Kp, Ki, Kd):
    from gops_b200 import _lib
    B = 1000
    rng = np.random.default_rng(int(Kp + 10 * Ki + Kd))
    state = torch.zeros(6, dtype=torch.float64, device="cuda")
    w = torch.zeros(3, dtype=torch.float32, device="cuda")
    ref = so.new_controller()
    seq = [(1000, 1000), (970, 990), (900, 950), (850, 700), (500, 960), (990, 1000), (0, 100)]
    seq += [tuple(rng.integers(0, B + 1, 2)) for _ in range(8)]
    for c0, c1 in seq:
        tail = torch.tensor([0.0, 0.0, float(c0), float(c1)], dtype=torch.float32, device="cuda")
        _lib.check(_lib.lib().gops_b200_spil_controller(_lib.ptr(tail), B, float(Kp), float(Ki), float(Kd), 0.97, 0.97,
                                                        _lib.ptr(state), _lib.ptr(w), _lib.stream_ptr()))
        sp = np.array([c0, c1], dtype=np.float32) / np.float32(B)
        w_r, w_c = so.spil_weights(ref, sp, Kp=Kp, Ki=Ki, Kd=Kd)
        st = state.cpu().numpy()
        np.testing.assert_array_equal(st[0:2], ref["delta_i"])
        np.testing.assert_array_equal(st[2:4], ref["safe_prob_pre"].astype(np.float64))
        np.testing.assert_array_equal(st[4:6], ref["lam"])
        np.testing.assert_array_equal(w.cpu().numpy(), np.array([w_r, *w_c], dtype=np.float32))


def test_launches_and_controller_trajectory():
    from gops_b200 import _lib
    from gops_b200.trainer.device_trainer import DeviceStateSampler
    torch.manual_seed(0)
    alg = _alg(2.0, 2.0)
    alg.loss_lag = 1
    sampler = DeviceStateSampler("pyth_veh3dofconti_errcstr", "cuda", 3, pre_horizon=10)
    alg.local_update(sampler.sample(4096), 0)          # warm-up: plans, scratch
    torch.cuda.synchronize()
    ref = so.new_controller()
    ref["delta_i"], ref["safe_prob_pre"], ref["lam"] = alg.delta_i, alg.safe_prob, alg.lam
    probs = []
    for it in range(1, 11):
        batch = sampler.sample(4096)
        n0 = _lib.lib().gops_b200_launch_count()
        tb = alg.local_update(batch, it)
        assert _lib.lib().gops_b200_launch_count() - n0 == LAUNCHES_PER_UPDATE
        assert all(math.isfinite(v) for v in tb.values())
        probs.append(alg.safe_prob)
    for sp in probs:
        so.spil_weights(ref, sp)
    np.testing.assert_array_equal(alg.lam, ref["lam"])
    np.testing.assert_array_equal(alg.delta_i, ref["delta_i"])


def test_refusals():
    from gops_b200 import _lib
    from gops_b200.create_pkg.create_alg import create_alg
    with pytest.raises(ValueError, match="pyth_veh3dofconti_errcstr"):
        _alg(env_id="pyth_veh3dofconti")
    with pytest.raises(ValueError, match="constraint_dim"):
        _alg(constraint_dim=3)
    # the kernel mode itself on a model without the constraint
    inf = create_alg(**_kwargs(env_id="pyth_veh3dofconti", algorithm="INFADP"))
    plan = inf._plan(_lib.ALG_INFADP_VALUE, inf.networks.policy, inf.networks.v, 10, 0.99)
    assert _lib.lib().gops_b200_plan_set_constraint(plan.handle, 4, 1.0) != 0
    assert b"pyth_veh3dofconti_errcstr" in _lib.lib().gops_b200_last_error()
    # no wgmma path for SPIL
    alg = _alg()
    alg.kernel_path = "tc"
    data = orc.sample_inputs("pyth_veh3dofconti", 256, seed=5, pre_horizon=10)
    with pytest.raises(RuntimeError, match="wgmma"):
        alg.local_update(data, 0)


def test_example_script_trains():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "example_train", "spil_mlp_veh3dofconti_errcstr_b200.py"),
                          "--max_iteration", "21", "--eval_interval", "10", "--log_save_interval", "5",
                          "--replay_batch_size", "1024"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    losses = [float(x) for line in out.stdout.splitlines() for x in
              [part.split(":")[1].strip(" }") for part in line.split(",") if "loss-RL iter" in part]]
    assert len(losses) >= 8 and all(math.isfinite(x) for x in losses), out.stdout[-2000:]
