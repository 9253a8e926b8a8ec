"""CPU: the RPI oracle (oracle/rpi_oracle.py) against the unmodified reference (tests/golden/rpi_osc_*.npz), the hand
derivation of the Hamiltonian gradient that csrc/rpi.cu implements against autograd's double backward, the container's
state_dict keys and init law, and the configurations the RPI kernels refuse."""
import os

import numpy as np
import pytest
import torch

from golden_util import GOLDEN
from oracle import rpi_oracle as ro

CASES = {"rpi_osc_a": 64, "rpi_osc_b": 256, "rpi_osc_c": 64}
MAX_STEPS = {"rpi_osc_a": 10000, "rpi_osc_b": 10000, "rpi_osc_c": 3}


def load_rpi(name):
    rec = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    n_iter = sum(1 for k in rec if k.endswith("/n"))
    offs = rec["draw_offsets"]
    draws = [rec["draws"][offs[i]:offs[i + 1]] for i in range(n_iter)]
    sd0 = {k[len("init/"):]: rec[k] for k in rec if k.startswith("init/")}
    return rec, n_iter, draws, sd0


def replay(name, dtype):
    rec, n_iter, draws, sd0 = load_rpi(name)
    out, sd, adam, x, _ = ro.run(sd0, "elu", 2.0, rec["obs0"], rec["max_step"], draws, n_iter,
                                 max_steps=MAX_STEPS[name], dtype=dtype)
    return rec, n_iter, out, adam, x


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_replays_the_reference(name, dtype):
    torch.set_num_threads(4)
    rec, n_iter, out, adam, x = replay(name, dtype)
    assert [o["n"] for o in out] == [int(rec[f"it{i}/n"]) for i in range(n_iter)]
    for i, o in enumerate(out):
        assert rel(o["loss"], rec[f"it{i}/loss"]) < 1e-4
        assert rel(o["h_after"], rec[f"it{i}/h_after"]) < 1e-4
        assert abs(o["h_before"] - rec[f"it{i}/h_before"]) <= 1e-4 * abs(rec[f"it{i}/h_before"])
        assert rel(o["flat"], rec[f"it{i}/flat"]) < 1e-4
    assert rel(adam[0], rec["adam/exp_avg"]) < 1e-3
    assert rel(adam[1], rec["adam/exp_avg_sq"]) < 1e-3
    np.testing.assert_allclose(x, rec["final_obs"], atol=1e-4)


@pytest.mark.parametrize("act", ["relu", "elu", "gelu", "selu", "sigmoid", "tanh"])
def test_hand_derivation_matches_double_backward(act):
    g = torch.Generator().manual_seed(11)
    sd = {k: (torch.rand(s, generator=g, dtype=torch.float64) - 0.5) * sc for k, s, sc in
          zip(ro.KEYS, [(64, 2), (64,), (64, 64), (64,), (1, 64), (1,)], [1.5, 0.4, 0.5, 0.4, 0.6, 0.2])}
    x = (torch.rand(128, 2, generator=g, dtype=torch.float64) - 0.5) * 4
    aw = (torch.rand(128, 2, generator=g, dtype=torch.float64) - 0.5) * 3
    value = ro.Value(sd, act, torch.float64)
    loss, grad = ro.loss_and_grad(value, x, aw, 2.0)
    f, c = ro.wrapped_model(x, aw, 2.0)
    l2, g2 = ro.hand_loss_grad({k: v.numpy() for k, v in sd.items()}, act, x.numpy(), f.numpy(), c.numpy())
    assert abs(l2 - loss.item()) < 1e-12 * max(1.0, abs(l2))
    np.testing.assert_allclose(g2, grad.numpy(), rtol=1e-9, atol=1e-12)


def rpi_kwargs(**over):
    kw = dict(env_id="pyth_oscillatorconti", algorithm="RPI", trainer="on_serial_trainer", seed=0, is_adversary=True,
              value_func_name="StateValue", value_func_type="MLP", value_hidden_sizes=[64, 64],
              value_hidden_activation="elu", value_output_activation="linear", policy_func_name="DetermPolicy",
              policy_func_type="POLY", policy_act_distribution="default", learning_rate=1e-3, gamma_atte=2.0,
              max_newton_iteration=50, max_step_update_value=10000, reset_batch_size=64, sample_batch_size=64,
              fixed_initial_state=[0.5, -0.5], initial_state_range=[1.2, 1.2], state_threshold=[5.0, 5.0],
              lower_step=100, upper_step=200, obsv_dim=2, action_dim=1, action_type="continu",
              action_high_limit=np.ones(1, np.float32), action_low_limit=-np.ones(1, np.float32))
    kw.update(over)
    return kw


def test_state_dict_keys_and_init_law():
    from gops_b200.create_pkg.create_alg import create_alg
    rec, _, _, sd0 = load_rpi("rpi_osc_a")
    torch.manual_seed(int(rec["seed"]))
    np.random.seed(int(rec["seed"]))
    alg = create_alg(**rpi_kwargs(seed=int(rec["seed"])))
    keys = [f"{n}.{k}" for n in ("value", "value_target") for k in ro.KEYS]
    assert list(alg.networks.state_dict().keys()) == keys
    sd = alg.networks.state_dict()
    for k in ro.KEYS:      # Xavier-uniform weights and zero biases, drawn in the reference's order
        np.testing.assert_array_equal(sd["value." + k].numpy(), sd0[k])
        np.testing.assert_array_equal(sd["value_target." + k].numpy(), sd0[k])
    # the sampler's first reset and the episode caps come from the model's NumPy draws, as in the reference
    np.testing.assert_array_equal(alg.obs.numpy(), rec["obs0"])
    np.testing.assert_array_equal(alg.max_step_per_episode.numpy(), np.floor(rec["max_step"]))


@pytest.mark.parametrize("over,exc,match", [
    (dict(is_adversary=False), ValueError, "is_adversary"),
    (dict(value_func_type="POLY"), NotImplementedError, "MLP"),
    (dict(value_hidden_sizes=[256, 256]), NotImplementedError, r"\[64, 64\]"),
    (dict(value_hidden_sizes=[64, 32]), NotImplementedError, r"\[64, 64\]"),
    (dict(reset_batch_size=96), ValueError, "multiple of 64"),
    (dict(reset_batch_size=576), ValueError, "at most 512"),
])
def test_refusals(over, exc, match):
    from gops_b200.create_pkg.create_alg import create_alg
    with pytest.raises(exc, match=match):
        create_alg(**rpi_kwargs(**over))


def test_refuses_more_than_one_rank(monkeypatch):
    import torch.distributed as dist
    from gops_b200.algorithm import rpi
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda: 2)
    with pytest.raises(NotImplementedError, match="one GPU"):
        rpi.check_config(**rpi_kwargs())
