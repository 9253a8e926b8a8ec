"""CPU: the approximate-function containers of DSAC, DSAC-T, SAC, INFADP and SPIL -- state_dict keys in the reference
container's order (a checkpoint written by either loads into the other), the adjustable parameters and optimizers of
each algorithm, and Polyak targets that own their flat parameter storage (a target's update never writes into the
network it follows)."""
import importlib

import numpy as np
import pytest
import torch

from oracle import ref_shim

needs_reference = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not reachable")

_COMMON = dict(seed=0, trainer="off_serial_trainer", cnn_shared=False, action_type="continu",
               policy_func_type="MLP", value_func_type="MLP", policy_output_activation="linear",
               value_output_activation="linear")
_SOFT_AC = dict(env_id="pyth_idpendulum", obsv_dim=6, action_dim=1, action_high_limit=np.ones(1, np.float32),
                action_low_limit=-np.ones(1, np.float32), policy_func_name="StochaPolicy",
                policy_hidden_sizes=[64, 64, 64], policy_hidden_activation="gelu",
                policy_act_distribution="TanhGaussDistribution", policy_min_log_std=-20, policy_max_log_std=1,
                value_hidden_sizes=[64, 64, 64], value_hidden_activation="gelu", value_learning_rate=3e-4,
                policy_learning_rate=3e-4, alpha_learning_rate=5e-3, gamma=0.99, tau=0.005, auto_alpha=True,
                alpha=0.2)
_ADP = dict(env_id="pyth_veh3dofconti_errcstr", obsv_dim=46, action_dim=2, action_high_limit=np.ones(2, np.float32),
            action_low_limit=-np.ones(2, np.float32), policy_func_name="DetermPolicy", policy_hidden_sizes=[64, 64],
            policy_hidden_activation="relu", policy_act_distribution="default", policy_learning_rate=1e-3,
            value_func_name="StateValue", value_hidden_sizes=[64, 64], value_hidden_activation="relu",
            value_learning_rate=1e-3, pre_horizon=10, forward_step=10, constraint_dim=2, gamma=0.99, tau=0.005)

# algorithm: (kwargs, adjustable_parameters, optimizer_dict keys, (network, its Polyak target) pairs)
CASES = {
    "DSAC": (dict(_SOFT_AC, value_func_name="ActionValueDistri", delay_update=2, TD_bound=10, bound=True),
             ("gamma", "tau", "auto_alpha", "alpha", "bound", "delay_update"), ["q", "policy"],
             [("q", "q_target"), ("policy", "policy_target")]),
    "DSACT": (dict(_SOFT_AC, value_func_name="ActionValueDistri", delay_update=2),
              ("gamma", "tau", "auto_alpha", "alpha", "delay_update"), ["q1", "q2", "policy"],
              [("q1", "q1_target"), ("q2", "q2_target"), ("policy", "policy_target")]),
    "SAC": (dict(_SOFT_AC, value_func_name="ActionValue", q_learning_rate=3e-4),
            ("gamma", "tau", "auto_alpha", "alpha", "target_entropy"), ["q1", "q2", "policy"],
            [("q1", "q1_target"), ("q2", "q2_target")]),
    "INFADP": (dict(_ADP, env_id="pyth_veh3dofconti"),
               ("gamma", "tau", "pev_step", "pim_step", "forward_step", "reward_scale"), ["v", "policy"],
               [("v", "v_target"), ("policy", "policy_target")]),
    "SPIL": (dict(_ADP), ("gamma", "tau", "pev_step", "pim_step", "forward_step", "reward_scale"), ["v", "policy"],
             [("v", "v_target"), ("policy", "policy_target")]),
}


def _kwargs(name):
    return dict(_COMMON, algorithm=name, **CASES[name][0])


def _alg(name):
    from gops_b200.create_pkg.create_alg import create_alg
    torch.manual_seed(0)
    return create_alg(**_kwargs(name))


@needs_reference
@pytest.mark.parametrize("name", sorted(CASES))
def test_state_dict_keys_in_the_reference_order(name):
    ref_shim.install()
    module = {"DSACT": "dsact"}.get(name, name.lower())
    ref = importlib.import_module(f"gops.algorithm.{module}").ApproxContainer(**_kwargs(name))
    assert list(_alg(name).state_dict()) == list(ref.state_dict())


@pytest.mark.parametrize("name", sorted(CASES))
def test_parameters_optimizers_and_targets(name):
    _, adjustable, optimizers, pairs = CASES[name]
    alg = _alg(name)
    nets = alg.networks
    assert alg.adjustable_parameters == adjustable
    assert list(nets.optimizer_dict) == optimizers
    flats = [m.flat_params for m in nets.children() if hasattr(m, "flat_params")]
    assert len({id(f) for f in flats}) == len(flats) >= 2 * len(pairs)
    for src_name, tgt_name in pairs:
        src, tgt = getattr(nets, src_name), getattr(nets, tgt_name)
        fp = tgt.flat_params
        assert fp is not src.flat_params and any(m is fp.module for m in tgt.children()), tgt_name
        assert [id(p) for p in fp.module.parameters()] == [id(p) for p in tgt.parameters()], tgt_name
        assert not any(p.requires_grad for p in tgt.parameters()), tgt_name
        assert all(p.requires_grad for p in src.parameters()), src_name
        for a, b in zip(src.state_dict().values(), tgt.state_dict().values()):
            assert torch.equal(a, b) and a.data_ptr() != b.data_ptr(), tgt_name
