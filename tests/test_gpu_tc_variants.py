"""The FHADP wgmma rollout kernel built with the default wrapper chain, one action and GELU fixed at compile time
(csrc/model_kernels.cuh, kTcGeluChain) against the one that reads the wrapper flags at run time (kTcGelu).  An identity
ScaleObservation (scale 1, shift 0) moves an idpendulum plan from the first to the second without changing any value:
x / 1 - 0 and (x + 0) * 1 are exact, so loss and gradient must agree bit for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _loss_and_grad(**extra):
    from gops_b200.create_pkg.create_alg import create_alg
    from gops_b200.trainer import device_sampler as ds
    kw = dict(env_id="pyth_idpendulum", algorithm="FHADP", seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=6, action_dim=1, action_high_limit=np.ones(1, np.float32),
              action_low_limit=-np.ones(1, np.float32), policy_func_name="FiniteHorizonPolicy",
              policy_func_type="MLP", policy_hidden_sizes=[64, 64], policy_hidden_activation="gelu",
              policy_act_distribution="default", policy_learning_rate=1e-4, value_func_type="MLP", pre_horizon=12,
              reward_scale=1.0)
    kw.update(extra)
    torch.manual_seed(0)
    alg = create_alg(**kw)
    alg.kernel_path = "tc"
    data = ds.sample_idpendulum(3000, "cuda", 7)
    data["done"][::97] = 1.0
    alg._compute_gradient(data)
    grad = np.concatenate([p.grad.detach().cpu().numpy().ravel() for p in alg.networks.policy.parameters()])
    assert alg.last_kernel_path() == "tc"
    return {k: v for k, v in alg.tb_info.items() if "time" not in k.lower()}, grad


def test_fixed_chain_kernel_matches_runtime_flags_kernel():
    info_a, g_a = _loss_and_grad()
    info_b, g_b = _loss_and_grad(obs_scale=np.ones(6, np.float32), obs_shift=np.zeros(6, np.float32))
    assert np.any(g_a != 0) and info_a
    assert g_a.tobytes() == g_b.tobytes()
    assert info_a == info_b
