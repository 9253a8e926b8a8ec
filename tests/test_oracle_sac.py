"""CPU: oracle/sac_ref.py, replaying the recorded noise through the live unmodified reference, reproduces the recorded
SAC runs (tests/golden/sac_idp*.npz and the update of ckpt_sac_idp.npz, made by oracle/make_golden_sac.py) exactly:
tb values, gradients and post-update weights of every update (the weights as sac_ref.expand_golden rebuilds them; for
the shipped checkpoint the float64 sum and norm of every gradient tensor)."""
import numpy as np
import pytest
import torch

from golden_util import load
from oracle import ref_shim, sac_ref

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not reachable")


def _data(rec):
    return {k[3:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith("in_")}


def _check(rec, it, tb, grads, sd=None):
    want_tb = {k.split("/tb/")[1]: float(v) for k, v in rec.items() if k.startswith(f"it{it}/tb/")}
    assert len(want_tb) == 6 and tb == want_tb, (it, tb, want_tb)
    want_g = {k.split("/grad/")[1]: v for k, v in rec.items() if k.startswith(f"it{it}/grad/")}
    assert sorted(grads) == sorted(want_g), it
    for k, v in want_g.items():
        assert np.array_equal(grads[k], v), (it, k)
    if sd is not None:
        want_sd = {k.split("/post/")[1]: v for k, v in rec.items() if k.startswith(f"it{it}/post/")}
        assert sorted(sd) == sorted(want_sd), it
        for k, v in want_sd.items():
            assert np.array_equal(sd[k], v), (it, k)


@pytest.mark.parametrize("name", sorted(sac_ref.GOLDEN_CASES))
def test_sac_ref_reproduces_the_recorded_updates(name):
    torch.set_num_threads(4)
    n_iter, _, over = sac_ref.GOLDEN_CASES[name]
    kw = sac_ref.kwargs(**over)
    rec = sac_ref.expand_golden(load(name), kw)
    assert 1 + max(int(k[2:k.index("/")]) for k in rec if k.startswith("it")) == n_iter
    alg = sac_ref.create(kw, {k[5:]: v for k, v in rec.items() if k.startswith("init/")})
    data = _data(rec)
    for it in range(n_iter):
        tb, grads, sd = sac_ref.update(alg, data, rec[f"it{it}/eps_new"], rec[f"it{it}/eps_next"], it)
        _check(rec, it, tb, grads, sd)
        assert ("log_alpha" in grads) == over.get("auto_alpha", True)
    assert torch.equal(data["obs"], torch.from_numpy(rec["in_obs"]))      # the caller's batch is left as it was


def test_sac_ref_reproduces_the_update_from_the_shipped_checkpoint():
    torch.set_num_threads(4)
    rec = load("ckpt_sac_idp")
    assert sac_ref.checkpoint_sha256() == str(rec["ckpt_sha256"])
    c = sac_ref.CKPT
    alg = sac_ref.create(sac_ref.kwargs(c["hidden"], c["act"]), torch.load(sac_ref.checkpoint_path(), map_location="cpu"))
    tb, grads, _ = sac_ref.update(alg, _data(rec), rec["it0/eps_new"], rec["it0/eps_next"], 0)
    want_tb = {k.split("/tb/")[1]: float(v) for k, v in rec.items() if k.startswith("it0/tb/")}
    assert len(want_tb) == 6 and tb == want_tb, (tb, want_tb)
    keys = sorted(k.split("/grad_sum/")[1] for k in rec if k.startswith("it0/grad_sum/"))
    assert keys == sorted(k for k in grads if k != "log_alpha")
    assert np.array_equal(grads["log_alpha"], rec["it0/grad/log_alpha"])
    for k in keys:
        g = grads[k].astype(np.float64)
        assert g.sum() == rec[f"it0/grad_sum/{k}"] and np.linalg.norm(g) == rec[f"it0/grad_norm/{k}"], k
