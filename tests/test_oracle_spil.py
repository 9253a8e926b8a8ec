"""CPU: the oracle's SPIL restatement (oracle/spil_oracle.py) against the unmodified reference (tests/golden/spil_*.npz:
four consecutive updates on one pyth_veh3dofconti_errcstr batch, safe probability near and far from the chance
threshold), and a table test of the PI multiplier controller over synthetic safe-probability sequences."""
import numpy as np
import pytest
import torch

from golden_util import inputs_from, load, net_from, rel_l2
from oracle import gops_oracle as orc
from oracle import spil_oracle as so

TOLS = {"spil_near": (3.0, 2.3), "spil_far": (0.9, 1.6)}      # (y_error_tol, u_error_tol) of oracle/make_golden_spil.py


def _tb(rec, it, name):
    return float(rec[f"it{it}/tb/{name}-RL iter"])


@pytest.mark.parametrize("name", sorted(TOLS))
def test_oracle_follows_the_reference_over_four_updates(name):
    torch.set_num_threads(4)
    rec = load(name)
    y_tol, u_tol = TOLS[name]
    env = orc.create_env_model("pyth_veh3dofconti_errcstr", pre_horizon=10, y_error_tol=y_tol, u_error_tol=u_tol)
    data = inputs_from(rec, "pyth_veh3dofconti")
    ctl = so.new_controller()
    for it in range(4):
        prefix = "init/" if it == 0 else f"it{it - 1}/post/"
        v = net_from(rec, prefix, "v", "relu", requires_grad=True)
        vt = net_from(rec, prefix, "v_target", "relu")
        pol = net_from(rec, prefix, "policy", "relu", requires_grad=True)
        loss_v, vmean, issafe = so.spil_loss_value(v, pol, vt, env, data, 10, 0.99)
        loss_v.backward()
        ref = _tb(rec, it, "Loss/Critic loss")
        assert abs(loss_v.item() - ref) <= 2e-6 * max(1.0, abs(ref)), (it, loss_v.item(), ref)
        assert abs(vmean.item() - _tb(rec, it, "Train/Critic avg value")) <= 2e-6 * max(1.0, abs(vmean.item()))
        keys = [f"it{it}/grad/v.v.{2 * j}.{w}" for j in range(3) for w in ("weight", "bias")]
        assert rel_l2([t.grad.numpy() for pair in v.layers for t in pair], [rec[k] for k in keys]) < 1e-5
        sp = so.safe_probability(issafe)
        assert np.array_equal(sp, rec[f"it{it}/safe_prob"]), (it, sp, rec[f"it{it}/safe_prob"])
        w_r, w_c = so.spil_weights(ctl, sp)
        assert np.array_equal(ctl["lam"], rec[f"it{it}/lam"]) and np.array_equal(ctl["delta_i"], rec[f"it{it}/delta_i"])
        for p in pol.params():
            p.grad = None
        loss_pi = so.spil_loss_policy(pol, env, data, 10, 0.99, w_r, w_c)
        loss_pi.backward()
        ref = _tb(rec, it, "Loss/Actor loss")
        assert abs(loss_pi.item() - ref) <= 2e-6 * max(1.0, abs(ref)), (it, loss_pi.item(), ref)
        keys = [f"it{it}/grad/policy.pi.{2 * j}.{w}" for j in range(3) for w in ("weight", "bias")]
        assert rel_l2([t.grad.numpy() for pair in pol.layers for t in pair], [rec[k] for k in keys]) < 1e-5


def test_golden_settings_cover_both_controller_regimes():
    """near: every |chance_thre - safe_prob| <= 0.1 with lam > 0; far: every gap > 0.2 (the separated integral)."""
    near, far = load("spil_near"), load("spil_far")
    for it in range(4):
        gap = 0.97 - near[f"it{it}/safe_prob"].astype(np.float64)
        assert near[f"it{it}/safe_prob"][0] < 0.97 and near[f"it{it}/lam"][0] > 0.0 and np.all(np.abs(gap) <= 0.1)
        assert np.all(0.97 - far[f"it{it}/safe_prob"].astype(np.float64) > 0.2) and np.all(far[f"it{it}/lam"] > 0.0)


# (safe-prob sequence, Kp, Ki, Kd, initial delta_i): every branch of __spil_get_weight -- the separation at 0.1 and 0.2,
# the clips of delta_i at 0 and 99999, of delta_d and lam at 0 and 3333, and a non-zero Kd
CONTROLLER_TABLE = {
    "pi_band": ([0.95, 0.92, 0.9, 0.88], 60, 0.02, 0, 0.0),
    "separation_07": ([0.85, 0.82, 0.8], 60, 0.02, 0, 0.0),
    "separation_off": ([0.5, 0.6, 0.7, 0.76], 60, 0.02, 0, 0.0),
    "delta_i_clip_0": ([1.0, 0.99, 1.0], 60, 0.02, 0, 0.0),
    "delta_i_clip_99999": ([0.9, 0.91], 60, 0.02, 0, 99998.95),
    "lam_clip_3333": ([0.0, 0.1], 6000, 0.02, 0, 0.0),
    "lam_clip_0": ([1.0, 1.0], 60, 0.02, 0, 0.0),
    "kd_nonzero": ([0.9, 0.8, 0.85, 0.7, 0.95], 60, 0.02, 0.5, 0.0),
    "kd_large_lam_clip": ([0.95, 0.3, 0.9], 60, 0.02, 1e4, 0.0),
}


def _reference_controller(state, safe_prob, Kp, Ki, Kd):
    """Independent float64 / float32 statement of the controller step (the dtypes NumPy gives the reference)."""
    dp = 0.97 - safe_prob.astype(np.float64)
    sep = np.array([0.0 if abs(x) > 0.2 else (x * 0.7 if abs(x) > 0.1 else x) for x in dp])
    di = np.minimum(np.maximum(state["delta_i"] + sep, 0.0), 99999.0)
    pre = state["safe_prob_pre"]
    dd = pre - safe_prob                       # float64 on the first step, float32 afterwards
    dd = np.minimum(np.maximum(dd, 0), 3333).astype(dd.dtype)
    kd_dd = (np.float32(Kd) * dd) if dd.dtype == np.float32 else Kd * dd
    lam = np.minimum(np.maximum(Ki * di + Kp * dp + kd_dd.astype(np.float64), 0.0), 3333.0)
    return di, lam


@pytest.mark.parametrize("case", sorted(CONTROLLER_TABLE))
def test_controller_table(case):
    seq, Kp, Ki, Kd, di0 = CONTROLLER_TABLE[case]
    ctl = so.new_controller()
    ctl["delta_i"] = np.array([di0, 0.0])
    mirror = {k: v.copy() for k, v in ctl.items()}
    hit = set()
    for s in seq:
        sp = np.array([s, min(1.0, s + 0.05)], dtype=np.float32)
        dp = 0.97 - sp.astype(np.float64)
        hit |= {"sep_0.2" if abs(x) > 0.2 else ("sep_0.1" if abs(x) > 0.1 else "band") for x in dp}
        w_r, w_c = so.spil_weights(ctl, sp, Kp=Kp, Ki=Ki, Kd=Kd)
        di, lam = _reference_controller(mirror, sp, Kp, Ki, Kd)
        mirror.update(delta_i=di, lam=lam, safe_prob_pre=sp)
        assert np.array_equal(ctl["delta_i"], di) and np.array_equal(ctl["lam"], lam), (case, ctl, di, lam)
        assert w_r == 1 / (1 + lam.sum()) and np.array_equal(w_c, lam / (1 + lam.sum()))
        hit |= {"di_0" for x in di if x == 0.0} | {"di_max" for x in di if x == 99999.0}
        hit |= {"lam_0" for x in lam if x == 0.0} | {"lam_max" for x in lam if x == 3333.0}
    expected = {"pi_band": {"band"}, "separation_07": {"sep_0.1"}, "separation_off": {"sep_0.2"},
                "delta_i_clip_0": {"di_0", "lam_0"}, "delta_i_clip_99999": {"di_max"}, "lam_clip_3333": {"lam_max"},
                "lam_clip_0": {"lam_0"}, "kd_nonzero": {"band", "sep_0.1", "sep_0.2"},
                "kd_large_lam_clip": {"lam_max"}}[case]
    assert expected <= hit, (case, hit)
