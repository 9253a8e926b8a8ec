"""wgmma inference path (gops_b200/csrc/mlp_tc.cuh) against a float64 torch evaluation of the same
nn.Sequential (reference gops/apprfunc/mlp.py:73-77,103-111,327-329) and against the mma.sync path.
Tolerance: 3xTF32 keeps ~2^-21 per product; outputs are O(1), so 5e-6 absolute / 1e-5 relative."""
import copy
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref64(net, obs, virtual_t, squash):
    seq = copy.deepcopy(getattr(net, net._net_attr)).cpu().double()
    x = obs.double()
    if getattr(net, "_time_input", False):
        x = torch.cat([x, torch.full((x.shape[0], 1), float(virtual_t), dtype=torch.float64)], 1)
    y = seq(x)
    if squash:
        hi, lo = net.act_high_lim.double().cpu(), net.act_low_lim.double().cpu()
        y = (hi - lo) / 2 * torch.tanh(y) + (hi + lo) / 2
    return y.detach()


def _run(net, obs, mode, *args):
    old = os.environ.get("GOPS_B200_INFER")
    os.environ["GOPS_B200_INFER"] = mode
    try:
        out = net(obs, *args)
        torch.cuda.synchronize()
    finally:
        if old is None:
            os.environ.pop("GOPS_B200_INFER", None)
        else:
            os.environ["GOPS_B200_INFER"] = old
    return out.detach().cpu()


CASES = [
    # kind, obs_dim, act_dim, hidden activation
    ("finite", 6, 1, "gelu"),
    ("determ", 4, 2, "relu"),
    ("determ", 46, 2, "elu"),
    ("value", 6, 1, "tanh"),
    ("finite", 13, 2, "gelu"),
]


@pytest.mark.parametrize("kind,obs_dim,act_dim,act", CASES)
@pytest.mark.parametrize("B", [1, 127, 128, 129, 5000, 70001])
def test_tc_inference_matches_fp64_and_mma(kind, obs_dim, act_dim, act, B):
    from gops_b200.apprfunc.mlp import DetermPolicy, FiniteHorizonPolicy, StateValue
    torch.manual_seed(obs_dim * 1000 + B)
    kw = dict(obs_dim=obs_dim, act_dim=act_dim, hidden_sizes=(64, 64), hidden_activation=act,
              output_activation="linear", action_distribution_cls=None, act_high_lim=np.linspace(1.0, 2.0, act_dim).astype(np.float32),
              act_low_lim=-np.linspace(0.5, 1.5, act_dim).astype(np.float32))
    cls = {"finite": FiniteHorizonPolicy, "determ": DetermPolicy, "value": StateValue}[kind]
    net = cls(**kw).cuda()
    obs = torch.randn(B, obs_dim) * 1.5
    args = (7,) if kind == "finite" else ()
    ref = _ref64(net, obs, 7, kind != "value")
    if kind == "value":
        ref = ref.squeeze(-1)
    tc = _run(net, obs.cuda(), "tc", *args)
    mma = _run(net, obs.cuda(), "mma", *args)
    assert tc.shape == mma.shape == ref.shape
    np.testing.assert_allclose(tc.double().numpy(), ref.numpy(), rtol=1e-5, atol=5e-6)
    np.testing.assert_allclose(tc.numpy(), mma.numpy(), rtol=1e-5, atol=5e-6)
