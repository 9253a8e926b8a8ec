"""GPU: RPI's kernels (csrc/rpi.cu) against the fp64 oracle (oracle/rpi_oracle.py) and the unmodified reference
(tests/golden/rpi_osc_*.npz): the target policy at any batch, the single-step Hamiltonian loss and gradient for every
hidden activation, the Newton-iteration launch capped at one step against the single step plus FusedAdam (bit for bit),
whole Newton iterations replaying the reference's draws (exact inner-step counts), clusters of 4 and 8 CTAs,
determinism, one launch per Newton iteration, and the example script's checkpoint."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from golden_util import ROOT
from oracle import rpi_oracle as ro
from test_oracle_rpi import MAX_STEPS, load_rpi, rel, rpi_kwargs

pytestmark = pytest.mark.gpu

# oracle fp32-vs-fp64 spread on the same case (traces, weights) x 10: rpi_osc_a 2.1e-7 / 3.8e-7, rpi_osc_c 8.2e-8 /
# 1.2e-7 (measured with tests/test_oracle_rpi.replay)
BARS = {"rpi_osc_a": (2e-6, 4e-6), "rpi_osc_b": (2e-6, 4e-6), "rpi_osc_c": (1e-6, 2e-6)}


def make_alg(**over):
    from gops_b200 import _lib
    from gops_b200.create_pkg.create_alg import create_alg
    torch.manual_seed(0)
    np.random.seed(0)
    alg = create_alg(**rpi_kwargs(**over))
    alg.networks.cuda()
    _lib.lib()
    return alg


def set_value(alg, sd):
    with torch.no_grad():
        for net in (alg.networks.value, alg.networks.value_target):
            for (k, p) in zip(ro.KEYS, net.parameters()):
                p.copy_(torch.as_tensor(np.asarray(sd[k]), dtype=torch.float32))


def random_sd(seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return {k: ((torch.rand(s, generator=g) - 0.5) * sc * scale).numpy() for k, s, sc in
            zip(ro.KEYS, [(64, 2), (64,), (64, 64), (64,), (1, 64), (1,)], [1.5, 0.4, 0.5, 0.4, 0.6, 0.2])}


@pytest.mark.parametrize("B", [64, 100003])
def test_policy_matches_fp64_oracle(B):
    alg = make_alg()
    sd = random_sd(1)
    set_value(alg, sd)
    x = (torch.rand(B, 2, generator=torch.Generator().manual_seed(2)) - 0.5) * 4
    got = alg.networks.action_and_adversary(x.cuda()).cpu().double()
    ref = ro.action_and_adversary(ro.Value(sd, "elu", torch.float64), x.double(), 2.0)
    err = (got - ref).abs().max().item()
    assert err <= 2e-5 * max(1.0, ref.abs().max().item()), err
    assert torch.equal(alg.networks.policy(x[:64].cuda()).cpu(), got[:64, :1].float())


@pytest.mark.parametrize("act", ["relu", "elu", "gelu", "selu", "sigmoid", "tanh"])
@pytest.mark.parametrize("B", [64, 128, 512])
def test_single_step_loss_and_grad(act, B):
    alg = make_alg(value_hidden_activation=act)
    sd = random_sd(3)
    set_value(alg, sd)
    g = torch.Generator().manual_seed(B)
    x = (torch.rand(B, 2, generator=g) - 0.5) * 4
    aw = (torch.rand(B, 2, generator=g) - 0.5) * 3          # beyond [-1, 1]: the wrapper clips
    loss = alg.loss_and_grad(x, aw).item()
    grad = alg.networks.value.flat_params.gbuf[:4417].cpu().double().numpy()
    l64, g64 = ro.loss_and_grad(ro.Value(sd, act, torch.float64), x.double(), aw.double(), 2.0)
    assert abs(loss - l64.item()) <= 2e-6 * abs(l64.item())
    assert rel(grad, g64.numpy()) < 2e-5


def newton(alg, draws, max_steps=None, trace=True):
    if max_steps is not None:
        alg.max_step_update_value = max_steps
    alg.reset_override = torch.as_tensor(np.asarray(draws))
    alg.record_trace = trace
    return alg.local_update(None, 0)


def test_one_step_launch_is_single_step_plus_fused_adam():
    a1, a2 = make_alg(), make_alg()
    sd = random_sd(5)
    set_value(a1, sd)
    set_value(a2, sd)
    draws = (torch.rand(2, 64, 2, generator=torch.Generator().manual_seed(6)) - 0.5) * 2.4
    x0 = a1.obs.clone()
    newton(a1, draws, max_steps=1)
    aw = a2.networks.action_and_adversary(x0.cuda())
    a2.approximate_optimizer.zero_grad()
    a2.loss_and_grad(x0, aw)
    a2.approximate_optimizer.step()
    assert torch.equal(a1.networks.value.flat_params.flat, a2.networks.value.flat_params.flat)
    assert torch.equal(a1.approximate_optimizer._m, a2.approximate_optimizer._m)
    assert torch.equal(a1.approximate_optimizer._v, a2.approximate_optimizer._v)
    assert torch.equal(a1.networks.value_target.flat_params.flat, a1.networks.value.flat_params.flat)
    assert a1.approximate_optimizer._step == a2.approximate_optimizer._step == 1


@pytest.mark.parametrize("name", ["rpi_osc_a", "rpi_osc_b", "rpi_osc_c"])
def test_newton_iterations_follow_the_reference(name):
    rec, n_iter, draws, sd0 = load_rpi(name)
    B = rec["obs0"].shape[0]
    cfg = eval(str(rec["config"]))          # the case's settings, written by oracle/make_golden_rpi.py
    over = dict(reset_batch_size=B, sample_batch_size=B, max_step_update_value=MAX_STEPS[name])
    if "rng" in cfg:
        over["initial_state_range"] = list(cfg["rng"])
    alg = make_alg(**over)
    set_value(alg, sd0)
    alg.obs = torch.as_tensor(rec["obs0"])
    alg.max_step_per_episode = torch.as_tensor(np.floor(rec["max_step"]))
    tr_bar, w_bar = BARS[name]
    for it in range(n_iter):
        newton(alg, draws[it])
        assert alg.num_update_value == int(rec[f"it{it}/n"]), it
        tr = alg.last_trace.cpu().double().numpy()
        assert rel(tr[:, 0], rec[f"it{it}/loss"]) < tr_bar, it
        assert rel(tr[:, 1], rec[f"it{it}/h_after"]) < tr_bar, it
        assert rel(alg.networks.value.flat_params.flat.cpu().numpy(), rec[f"it{it}/flat"]) < w_bar, it
    opt = alg.approximate_optimizer
    assert opt._step == int(rec["adam/step"])
    assert rel(opt._m.cpu().numpy(), rec["adam/exp_avg"]) < 10 * w_bar
    assert rel(opt._v.cpu().numpy(), rec["adam/exp_avg_sq"]) < 10 * w_bar
    np.testing.assert_allclose(alg.obs.cpu().numpy(), rec["final_obs"], atol=1e-5)


def test_cluster_of_eight_matches_oracle():
    B, n_iter = 512, 3
    alg = make_alg(reset_batch_size=B, sample_batch_size=B, lower_step=5, upper_step=40, initial_state_range=[3.0, 3.0])
    sd = {k: v.detach().cpu().numpy() for k, v in zip(ro.KEYS, alg.networks.value.parameters())}
    obs0, cap = alg.obs.numpy().copy(), alg.max_step_per_episode.numpy().copy()
    g = torch.Generator().manual_seed(9)
    draws = [((torch.rand(400, B, 2, generator=g) - 0.5) * 6).numpy() for _ in range(n_iter)]
    out, _, _, x, _ = ro.run(sd, "elu", 2.0, obs0, cap, draws, n_iter, dtype=torch.float64)
    for it in range(n_iter):
        newton(alg, draws[it])
        assert alg.num_update_value == out[it]["n"], it
        assert rel(alg.networks.value.flat_params.flat.cpu().numpy(), out[it]["flat"]) < 1e-5, it


def test_deterministic_and_one_launch_per_iteration():
    from gops_b200 import _lib
    lib = _lib.lib()
    flats = []
    for _ in range(2):
        alg = make_alg(reset_batch_size=256, sample_batch_size=256)
        alg.record_trace = False
        n0 = lib.gops_b200_launch_count()
        for it in range(3):
            alg.local_update(None, it)
        torch.cuda.synchronize()
        assert lib.gops_b200_launch_count() - n0 == 3
        flats.append((alg.networks.value.flat_params.flat.clone(), alg.obs.clone(), alg.approximate_optimizer._m.clone()))
    for a, b in zip(*flats):
        assert torch.equal(a, b)


def test_example_script_and_reference_checkpoint(tmp_path):
    from oracle import ref_shim
    r = subprocess.run([sys.executable, os.path.join(ROOT, "example_train", "rpi_mlp_oscillatorconti_b200.py"),
                        "--max_newton_iteration", "3", "--save_folder", str(tmp_path)], capture_output=True, text=True,
                       cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "Newton ite: 2" in r.stdout
    pkl = tmp_path / "apprfunc" / "apprfunc_2.pkl"
    sd = torch.load(pkl, map_location="cpu")
    if not ref_shim.available():
        pytest.skip("reference not available")
    ref_shim.install()
    from gops.algorithm.rpi import ApproxContainer as RefContainer
    ref_kw = rpi_kwargs()
    ref_kw.pop("algorithm")
    ref_kw["cnn_shared"] = False
    ref = RefContainer(**ref_kw)
    ref.load_state_dict(sd)
    x = torch.tensor([[0.5, -0.5], [1.0, 0.3]])
    ours = ro.Value({k: sd["value_target." + k].numpy() for k in ro.KEYS}, "elu", torch.float64)
    np.testing.assert_allclose(ref.action_and_adversary(x.clone()).detach().double().numpy(),
                               ro.action_and_adversary(ours, x.double(), 2.0).numpy(), rtol=1e-5, atol=1e-6)
