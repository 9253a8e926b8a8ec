"""Parity AT THE BASELINE SIZES, on the path the library picks by itself (no environment switch; the test asserts which
kernel ran through the plan's launch record): fused sm_90a update vs. the fp32 CPU oracle evaluated in chunks.

  C1  FHADP pyth_idpendulum   H=30  B=2^18 and a ragged 200 003          (wgmma kernel, many chunks per CTA)
  C2  INFADP pyth_veh3dofconti P=10 n=10 B=4096, PEV and PIM             (mma.sync kernel, 46 inputs)
  C3  FHADP veh3dof_tracking  P=H=60 [256,256] elu B=8192 (one GPU's shard of 65 536): layer-wise wgmma path
  C5  INFADP pyth_lq s4a2     n=10  B=2^16 (PEV, PIM) and 2^20 (PIM)     (wgmma kernel)

Bars: loss 1e-4 relative, gradient 2e-4 relative L2 (1e-3 for pyth_veh3dofconti, see test_gpu_parity.py), number of
samples done at the end of the rollout EQUAL.  The fp32 oracle is itself within 2e-6 / 1e-5 of the unmodified
reference (tests/test_oracle_vs_golden.py) and within 5e-7 / 6e-6 of fp64 at these sizes (SURVEY A.4).
"""
import numpy as np
import pytest
import torch

from golden_util import oracle_chunked, rel_l2
from oracle import gops_oracle as orc

pytestmark = pytest.mark.gpu

LOSS_RTOL, GRAD_RTOL = 1e-4, 2e-4


def _alg(env_id, algname, act, hid, obs_dim, act_dim, seed, **extra):
    from gops_b200.create_pkg.create_alg import create_alg
    kw = dict(env_id=env_id, algorithm=algname, seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=obs_dim, action_dim=act_dim,
              action_high_limit=np.ones(act_dim, dtype=np.float32), action_low_limit=-np.ones(act_dim, dtype=np.float32),
              policy_func_name="FiniteHorizonPolicy" if algname == "FHADP" else "DetermPolicy", policy_func_type="MLP",
              policy_hidden_sizes=[hid, hid], policy_hidden_activation=act, policy_act_distribution="default",
              policy_learning_rate=1e-3, value_func_name="StateValue", value_func_type="MLP",
              value_hidden_sizes=[hid, hid], value_hidden_activation=act, value_learning_rate=1e-3)
    kw.update(extra)
    torch.manual_seed(seed)
    return create_alg(**kw)


def _spec(mod, seq, act, policy):
    net = getattr(mod, seq)
    layers = [(net[j].weight.detach().cpu().clone().requires_grad_(True),
               net[j].bias.detach().cpu().clone().requires_grad_(True)) for j in (0, 2, 4)]
    hi = mod.act_high_lim.detach().cpu() if policy else None
    lo = mod.act_low_lim.detach().cpu() if policy else None
    return orc.NetSpec(layers, act, "linear", hi, lo, time_input=getattr(mod, "_time_input", False))


def _gpu_data(env_id, data):
    if env_id == "veh3dof_tracking":
        from gops_b200.env.env_gen_ocp.pyth_base import ContextState, State
        robot, reference, t0 = data["state"]
        data = dict(data)
        data["state"] = State(robot_state=robot, context_state=ContextState(reference=reference, t=t0))
    return data


def _check(alg, net, got_loss, ref_loss, ref_grads, grad_rtol, expect_path):
    torch.cuda.synchronize()
    assert alg.last_kernel_path() == expect_path, (alg.last_kernel_path(), expect_path)
    assert abs(got_loss - ref_loss) <= LOSS_RTOL * max(1.0, abs(ref_loss)), (got_loss, ref_loss)
    got_g = [p.grad.detach().cpu().numpy() for p in getattr(alg.networks, net).parameters()]
    err = rel_l2(got_g, [g.numpy() for g in ref_grads])
    assert err < grad_rtol, err
    return err


@pytest.mark.parametrize("B", [1 << 18, 200003])
def test_c1_fhadp_idpendulum_headline(B):
    H = 30
    alg = _alg("pyth_idpendulum", "FHADP", "gelu", 64, 6, 1, seed=B % 1000, pre_horizon=H, reward_scale=1.0)
    data = orc.sample_inputs("pyth_idpendulum", B, seed=17)
    data["done"][::1001] = 1.0                                   # a few samples arrive done
    pol = _spec(alg.networks.policy, "pi", "gelu", True)
    env = orc.create_env_model("pyth_idpendulum", reward_scale=1.0)

    def chunk_loss(d):
        trace = []
        loss = orc.fhadp_loss(pol, env, d, H, 1.0, trace=trace)
        return loss, trace[-1][3].float().mean()                 # fraction done at the end of the rollout
    ref_loss, ref_g, extras = oracle_chunked(chunk_loss, data, pol.params())
    alg._compute_gradient(data)
    _check(alg, "policy", alg.tb_info["Loss/Actor loss-RL iter"], ref_loss, ref_g, GRAD_RTOL, "tc")
    n_done = float(alg.networks.policy.flat_params.gbuf[-2])     # tail = [loss | v-mean | #done | pad]
    assert n_done == round(extras[0] * B), (n_done, extras[0] * B)


def test_c2_infadp_veh3dofconti_b4096():
    B, n = 4096, 10
    alg = _alg("pyth_veh3dofconti", "INFADP", "relu", 64, 46, 2, seed=2, pre_horizon=10)
    data = orc.sample_inputs("pyth_veh3dofconti", B, seed=23, pre_horizon=10)
    env = orc.create_env_model("pyth_veh3dofconti", pre_horizon=10)
    for it in (0, 1):
        pol = _spec(alg.networks.policy, "pi", "relu", True)
        vt = _spec(alg.networks.v_target, "v", "relu", False)
        if it == 0:
            v = _spec(alg.networks.v, "v", "relu", False)
            ref_loss, ref_g, _ = oracle_chunked(lambda d: orc.infadp_loss_value(v, pol, vt, env, d, n, 0.99)[0], data,
                                                v.params(), chunk=2048)
            net, tag = "v", "Loss/Critic loss-RL iter"
        else:
            ref_loss, ref_g, _ = oracle_chunked(lambda d: orc.infadp_loss_policy(pol, vt, env, d, n, 0.99), data,
                                                pol.params(), chunk=2048)
            net, tag = "policy", "Loss/Actor loss-RL iter"
        alg.get_remote_update_info(data, it)
        _check(alg, net, alg.tb_info[tag], ref_loss, ref_g, 1e-3, "mma")


def test_c3_fhadp_veh3dof_tracking_w256_b8192():
    B, H = 8192, 60
    alg = _alg("veh3dof_tracking", "FHADP", "elu", 256, 6 + 4 * H, 2, seed=3, pre_horizon=H)
    data = orc.sample_inputs("veh3dof_tracking", B, seed=29, pre_horizon=H)
    pol = _spec(alg.networks.policy, "pi", "elu", True)
    env = orc.create_env_model("veh3dof_tracking", pre_horizon=H)
    ref_loss, ref_g, _ = oracle_chunked(lambda d: orc.fhadp_loss(pol, env, d, H, 1.0), data, pol.params(), chunk=1024)
    gd = _gpu_data("veh3dof_tracking", data)
    alg._compute_gradient(gd)
    _check(alg, "policy", alg.tb_info["Loss/Actor loss-RL iter"], ref_loss, ref_g, GRAD_RTOL, "tc")
    g_tc = alg.networks.policy.flat_params.gbuf.clone()
    alg.kernel_path = "mma"                      # the fused FP32-FFMA kernel stays available as the A/B baseline
    alg._compute_gradient(gd)
    _check(alg, "policy", alg.tb_info["Loss/Actor loss-RL iter"], ref_loss, ref_g, GRAD_RTOL, "mma")
    g_mma = alg.networks.policy.flat_params.gbuf
    assert (g_tc[:-4] - g_mma[:-4]).norm() <= 2e-4 * g_mma[:-4].norm()


def test_layerwise_update_graph_replay_matches_eager():
    """The layer-wise update is captured into a CUDA graph the second time the same call (buffers + constants) is
    seen and replayed from the third on: replays must reproduce the eager launch sequence, follow new CONTENTS of the
    same buffers, and a call with other buffers must not go through the stale graph."""
    B, H = 640, 12
    alg = _alg("veh3dof_tracking", "FHADP", "elu", 256, 6 + 4 * H, 2, seed=4, pre_horizon=H)
    from gops_b200.env.env_gen_ocp.pyth_base import ContextState, State

    def resident(seed):
        d = orc.sample_inputs("veh3dof_tracking", B, seed=seed, pre_horizon=H)
        robot, reference, t0 = d["state"]
        return {"obs": d["obs"].cuda(), "done": d["done"].cuda(),
                "state": State(robot_state=robot.cuda(), context_state=ContextState(reference=reference.cuda(), t=t0))}

    d1, d2 = resident(41), resident(42)
    gbuf = lambda: alg.networks.policy.flat_params.gbuf
    out = []
    for _ in range(4):                       # eager, eager (key seen twice -> capture), replay, replay
        alg._compute_gradient(d1)
        out.append((gbuf().clone(), float(alg.tb_info["Loss/Actor loss-RL iter"])))
    for g, l in out[1:]:
        assert abs(l - out[0][1]) <= 1e-6 * abs(out[0][1])
        assert (g - out[0][0]).norm() <= 1e-6 * out[0][0].norm()
    alg._compute_gradient(d2)                # other buffers: eager again
    g2, l2 = gbuf().clone(), float(alg.tb_info["Loss/Actor loss-RL iter"])
    assert abs(l2 - out[0][1]) > 1e-4 * abs(l2)
    d1["obs"].copy_(d2["obs"])               # same buffers as the captured call, new contents: the replay reads them
    d1["done"].copy_(d2["done"])
    d1["state"].robot_state.copy_(d2["state"].robot_state)
    d1["state"].context_state.reference.copy_(d2["state"].context_state.reference)
    for _ in range(3):
        alg._compute_gradient(d1)
        assert abs(float(alg.tb_info["Loss/Actor loss-RL iter"]) - l2) <= 1e-6 * abs(l2)
        assert (gbuf() - g2).norm() <= 1e-6 * g2.norm()


@pytest.mark.parametrize("B,its", [(1 << 16, (0, 1)), (1 << 20, (1,))])
def test_c5_infadp_lq_sweep_ends(B, its):
    n = 10
    alg = _alg("pyth_lq", "INFADP", "gelu", 64, 4, 2, seed=5, lq_config="s4a2", reward_scale=1.0, reward_shift=0.0)
    data = orc.sample_inputs("pyth_lq", B, seed=31, lq_config="s4a2")
    env = orc.create_env_model("pyth_lq", lq_config="s4a2", reward_scale=1.0, reward_shift=0.0)
    for it in its:
        pol = _spec(alg.networks.policy, "pi", "gelu", True)
        vt = _spec(alg.networks.v_target, "v", "gelu", False)
        if it == 0:
            v = _spec(alg.networks.v, "v", "gelu", False)
            ref_loss, ref_g, _ = oracle_chunked(lambda d: orc.infadp_loss_value(v, pol, vt, env, d, n, 0.99)[0], data,
                                                v.params(), chunk=65536)
            net, tag = "v", "Loss/Critic loss-RL iter"
        else:
            ref_loss, ref_g, _ = oracle_chunked(lambda d: orc.infadp_loss_policy(pol, vt, env, d, n, 0.99), data,
                                                pol.params(), chunk=65536)
            net, tag = "policy", "Loss/Actor loss-RL iter"
        alg.get_remote_update_info(data, it)
        _check(alg, net, alg.tb_info[tag], ref_loss, ref_g, GRAD_RTOL, "tc")


def test_plan_path_option_is_explicit_and_assertable():
    """The kernel path is a plan option (gops_b200_plan_set_path), not only an environment switch: forcing 'tc' on a
    tiny batch and 'mma' on a large one both take effect and are reported by the launch record."""
    alg = _alg("pyth_idpendulum", "FHADP", "gelu", 64, 6, 1, seed=7, pre_horizon=5, reward_scale=1.0)
    small = orc.sample_inputs("pyth_idpendulum", 300, seed=1)
    alg.kernel_path = "tc"
    alg._compute_gradient(small)
    g_tc = alg.networks.policy.flat_params.gbuf.clone()
    assert alg.last_kernel_path() == "tc"
    alg.kernel_path = "mma"
    alg._compute_gradient(small)
    assert alg.last_kernel_path() == "mma"
    g_mma = alg.networks.policy.flat_params.gbuf
    assert (g_tc[:-4] - g_mma[:-4]).norm() <= 2e-4 * g_mma[:-4].norm()
    wide = _alg("pyth_veh3dofconti", "INFADP", "relu", 64, 46, 2, seed=2, pre_horizon=10)
    wide.kernel_path = "tc"
    with pytest.raises(RuntimeError, match="not built"):
        wide.get_remote_update_info(orc.sample_inputs("pyth_veh3dofconti", 64, seed=2, pre_horizon=10), 0)
