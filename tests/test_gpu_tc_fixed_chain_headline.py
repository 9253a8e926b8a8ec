"""The fixed-chain FHADP wgmma kernel (kTcGeluChain: layer 1 of the forward sweep and layer 2 of the reverse sweep fed
from registers) against the kernel that reads the wrapper flags at run time (kTcGelu: the reverse sweep reads both
layers' A operands from shared memory) at the headline horizon H = 30, with `done` set on some samples.  The identity ScaleObservation
selects the second kernel without changing any value, so loss and gradient must agree bit for bit.  The batches give
the warpgroup slots of an H100 (132 SMs x 3 warpgroups) two or three, and ten or eleven sub-tiles each, the first with
a ragged last sub-tile; so every slot runs reverse steps back to back, across sub-tiles as well."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _loss_and_grad(batch, **extra):
    from gops_b200.create_pkg.create_alg import create_alg
    from gops_b200.trainer import device_sampler as ds
    kw = dict(env_id="pyth_idpendulum", algorithm="FHADP", seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=6, action_dim=1, action_high_limit=np.ones(1, np.float32),
              action_low_limit=-np.ones(1, np.float32), policy_func_name="FiniteHorizonPolicy",
              policy_func_type="MLP", policy_hidden_sizes=[64, 64], policy_hidden_activation="gelu",
              policy_act_distribution="default", policy_learning_rate=1e-4, value_func_type="MLP", pre_horizon=30,
              reward_scale=1.0)
    kw.update(extra)
    torch.manual_seed(0)
    alg = create_alg(**kw)
    alg.kernel_path = "tc"
    data = ds.sample_idpendulum(batch, "cuda", 7)
    data["done"][::97] = 1.0
    alg._compute_gradient(data)
    grad = np.concatenate([p.grad.detach().cpu().numpy().ravel() for p in alg.networks.policy.parameters()])
    assert alg.last_kernel_path() == "tc"
    return {k: v for k, v in alg.tb_info.items() if "time" not in k.lower()}, grad


@pytest.mark.parametrize("batch", [(1 << 16) + 37, 1 << 18])
def test_fixed_chain_kernel_matches_runtime_flags_kernel_at_headline_horizon(batch):
    info_a, g_a = _loss_and_grad(batch)
    info_b, g_b = _loss_and_grad(batch, obs_scale=np.ones(6, np.float32), obs_shift=np.zeros(6, np.float32))
    assert np.any(g_a != 0) and info_a
    assert g_a.tobytes() == g_b.tobytes()
    assert info_a == info_b
