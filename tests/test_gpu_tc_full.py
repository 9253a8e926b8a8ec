"""wgmma rollout kernel (BF16x3 operands, FP32 weight-gradient accumulation; plan option kernel_path = "tc";
csrc/rollout_tc2.cuh) held to the same bars as the mma.sync kernel: golden vectors of the unmodified reference (loss,
gradient, Adam step), the fp64 oracle on ragged batches, degenerate shapes and the no-grad trace."""
import numpy as np
import pytest
import torch

import test_gpu_parity as base
from golden_util import CASES

pytestmark = pytest.mark.gpu

TC_GOLDEN = [n for n in base.GOLDEN
             if CASES[n][0] in ("pyth_idpendulum", "pyth_lq") and "w256" not in n]


@pytest.fixture(autouse=True)
def _force_tc(monkeypatch):
    """Every algorithm built in these tests asks its plans for the wgmma kernel (a plan option, asserted below)."""
    from gops_b200.algorithm.base import FusedADPMixin
    monkeypatch.setattr(FusedADPMixin, "kernel_path", "tc")


@pytest.mark.parametrize("name", TC_GOLDEN)
def test_tcf_golden_loss_grad_update(name):
    base.test_golden_loss_grad_update(name)


@pytest.mark.parametrize("env_id,algname,act,B,H,wk", base.oracle_cases([
    ("pyth_idpendulum", "FHADP", "gelu", 3000, 30),
    ("pyth_idpendulum", "FHADP", "tanh", 777, 7),
    ("pyth_idpendulum", "INFADP", "elu", 2048, 10),
    ("pyth_lq", "INFADP", "gelu", 5000, 10),
    ("pyth_lq", "FHADP", "selu", 1000, 25),
    ("pyth_lq", "INFADP", "sigmoid", 130, 3),
    ("pyth_idpendulum", "FHADP", "gelu", 1500, 10, "obs-rep3last-clip"),
]))
def test_tcf_against_oracle_fp64(env_id, algname, act, B, H, wk):
    base.test_against_oracle_fp64(env_id, algname, act, B, H, wk)


@pytest.mark.parametrize("B,H", [(1, 1), (1, 5), (17, 1), (129, 2), (513, 3)])
def test_tcf_edge_shapes(B, H):
    base.test_edge_shapes_against_oracle(B, H)


def test_tcf_trace_matches_reference_rollout():
    base.test_trace_matches_reference_rollout()


def test_tcf_path_is_taken_and_deterministic(monkeypatch):
    """Same inputs: hybrid and mma.sync gradients agree to tolerance but not bitwise (the wgmma forward rounds
    differently), and the hybrid path reproduces itself bit for bit."""
    alg, rec = base.build_alg("fhadp_idp_h30")
    data = base.data_from(rec, "pyth_idpendulum")

    def grads():
        alg._compute_gradient(data)
        torch.cuda.synchronize()
        return np.concatenate([p.grad.detach().cpu().numpy().ravel() for p in alg.networks.policy.parameters()])

    g_tc, g_tc2 = grads(), grads()
    assert alg.last_kernel_path() == "tc"
    alg.kernel_path = "mma"
    g_mma = grads()
    assert alg.last_kernel_path() == "mma"
    assert np.array_equal(g_tc, g_tc2)
    assert not np.array_equal(g_tc, g_mma)
    assert np.linalg.norm(g_tc - g_mma) <= 2e-4 * np.linalg.norm(g_mma)
