"""Constrained FHADP variants (N3: fhadp_exterior / fhadp_lagrangian / fhadp_interior on pyth_veh3dofconti_errcstr) on the
fused kernel (csrc/kernel.cuh cstr_mode 1 / 2 / 3) against the unmodified reference's golden vectors (two consecutive
updates: losses incl. the reward / constraint split, feasible ratio, gradients, the annealed penalty / learned multiplier)
and against the fp64 oracle on a fresh ragged batch with done samples (frozen observations keep paying the constraint)."""
import numpy as np
import pytest
import torch

from golden_util import inputs_from, load, oracle_chunked, rel_l2
from oracle import gops_oracle as orc

pytestmark = pytest.mark.gpu

EXTRA = {"FHADPExterior": dict(penalty=2.0, penalty_increase=1.5, penalty_delay=1),
         "FHADPInterior": dict(penalty=2.0, penalty_increase=1.5, penalty_delay=1),
         "FHADPLagrangian": dict(multiplier=1.5, multiplier_lr=5e-2, multiplier_delay=1)}
GRAD_RTOL = 1e-3        # pyth_veh3dofconti: fp32 finite-difference heading in the reference (see test_gpu_parity.py)


def _alg(algname, **over):
    from gops_b200.create_pkg.create_alg import create_alg
    kw = dict(env_id="pyth_veh3dofconti_errcstr", algorithm=algname, seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=46, action_dim=2, action_high_limit=np.ones(2, np.float32),
              action_low_limit=-np.ones(2, np.float32), policy_func_name="FiniteHorizonPolicy", policy_func_type="MLP",
              policy_hidden_sizes=[64, 64], policy_hidden_activation="elu", policy_act_distribution="default",
              policy_learning_rate=1e-3, value_func_type="MLP", pre_horizon=10, gamma=0.97, y_error_tol=1.2,
              u_error_tol=2.2)
    kw.update(EXTRA[algname])
    kw.update(over)
    return create_alg(**kw)


@pytest.mark.parametrize("algname", sorted(EXTRA))
def test_two_updates_follow_the_reference(algname):
    rec = load("cstr_" + algname.lower())
    alg = _alg(algname)
    alg.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("init/")})
    data = inputs_from(rec, "pyth_veh3dofconti")
    for it in (0, 1):
        if it == 1:
            alg.load_state_dict({k.split("/post/")[1]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("it0/post/")})
        tb = alg.local_update(data, it)
        for k in (k for k in rec if k.startswith(f"it{it}/tb/")):
            ref = float(rec[k])
            got = tb[k.split("/tb/")[1]]
            assert abs(got - ref) <= 1e-4 * max(1.0, abs(ref)), (it, k, got, ref)
        keys = sorted(k for k in rec if k.startswith(f"it{it}/grad/policy."))
        named = dict(alg.networks.policy.named_parameters())
        err = rel_l2([named[k.split("/grad/policy.")[1]].grad.cpu().numpy() for k in keys], [rec[k] for k in keys])
        bar = GRAD_RTOL
        if algname == "FHADPInterior":
            # the log barrier's gradient is 1 / c for constraints c -> 0-: a sample near the boundary amplifies fp32
            # round-off without bound.  Noise floor of THIS case = distance between the reference's own fp32 gradient
            # and the fp64 evaluation of the same formulas (1.7e-2 at the second update); the bar is three times that.
            from golden_util import net_from
            env64 = orc.create_env_model("pyth_veh3dofconti_errcstr", dtype=torch.float64, pre_horizon=10, y_error_tol=1.2,
                                         u_error_tol=2.2)
            pol64 = net_from(rec, "init/" if it == 0 else "it0/post/", "policy", "elu", torch.float64, requires_grad=True)
            pol64.time_input = True
            l64 = orc.fhadp_constrained_loss("interior", pol64, env64, inputs_from(rec, "pyth_veh3dofconti", torch.float64),
                                             10, 0.97, 2.0 * 1.5 ** it)[0]
            l64.backward()
            order = [f"it{it}/grad/policy.pi.{2 * j}.{w}" for j in range(3) for w in ("weight", "bias")]
            noise = rel_l2([t.grad.numpy() for pair in pol64.layers for t in pair], [rec[k] for k in order])
            bar = max(GRAD_RTOL, 3.0 * noise)
        assert err < bar, (it, err, bar)


@pytest.mark.parametrize("algname,mode", [("FHADPExterior", "exterior"), ("FHADPLagrangian", "lagrangian"),
                                          ("FHADPInterior", "interior")])
def test_against_fp64_oracle_with_done_samples(algname, mode):
    check_against_fp64_oracle(algname, mode, 777)


def check_against_fp64_oracle(algname, mode, B, seed=None):
    """test_against_fp64_oracle_with_done_samples at any batch size (the oracle runs in chunks of 32768 samples); the
    inputs are drawn with `seed` (default: B)."""
    torch.manual_seed(B)
    alg = _alg(algname, reward_scale=0.5)
    data = orc.sample_inputs("pyth_veh3dofconti", B, seed=B if seed is None else seed, pre_horizon=10)
    data["done"][::5] = 1.0
    env = orc.create_env_model("pyth_veh3dofconti_errcstr", dtype=torch.float64, pre_horizon=10, y_error_tol=1.2,
                               u_error_tol=2.2, reward_scale=0.5)
    pi = alg.networks.policy.pi
    layers = [(pi[j].weight.detach().cpu().double().requires_grad_(True), pi[j].bias.detach().cpu().double().requires_grad_(True))
              for j in (0, 2, 4)]
    pol = orc.NetSpec(layers, "elu", "linear", torch.ones(2, dtype=torch.float64), -torch.ones(2, dtype=torch.float64),
                      time_input=True)
    coef = 2.0 if mode != "lagrangian" else 1.5
    d64 = {k: (v.double() if v.is_floating_point() else v) for k, v in data.items()}
    loss, ref_g, (l_r, l_c, feas) = oracle_chunked(
        lambda d: orc.fhadp_constrained_loss(mode, pol, env, d, 10, 0.97, coef), d64, pol.params())
    tb = alg.get_remote_update_info(data, 0)[0]
    assert abs(tb["Loss/Actor loss-RL iter"] - loss) <= 1e-4 * max(1.0, abs(loss))
    assert abs(tb["Loss/Actor constraint loss-RL iter"] - l_c) <= 1e-4 * max(1.0, abs(l_c))
    bar = GRAD_RTOL
    if mode == "interior":
        assert abs(tb["Loss/Feasible ratio-RL iter"] - feas) < 1e-6
        # the log barrier amplifies the round-off of samples near the boundary (see above): noise floor = distance
        # between the fp32 and the fp64 evaluation of the same oracle on this batch; the bar is three times that
        env32 = orc.create_env_model("pyth_veh3dofconti_errcstr", dtype=torch.float32, pre_horizon=10, y_error_tol=1.2,
                                     u_error_tol=2.2, reward_scale=0.5)
        pol32 = orc.NetSpec([(w.detach().float().requires_grad_(True), b.detach().float().requires_grad_(True))
                             for w, b in layers], "elu", "linear", torch.ones(2), -torch.ones(2), time_input=True)
        _, g32, _ = oracle_chunked(lambda d: orc.fhadp_constrained_loss(mode, pol32, env32, d, 10, 0.97, coef), data,
                                   pol32.params())
        bar = max(GRAD_RTOL, 3.0 * rel_l2([g.numpy() for g in g32], [g.numpy() for g in ref_g]))
    got = [p.grad.detach().cpu().numpy() for p in alg.networks.policy.parameters()]
    err = rel_l2(got, [g.numpy() for g in ref_g])
    print(f"{algname} B={B}: gradient rel. L2 {err:.2e} (bar {bar:.2e})")
    assert err < bar, (err, bar)
