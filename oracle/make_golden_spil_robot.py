"""Generate tests/golden/spil_robot.npz and tests/golden/ckpt_spil_robot.npz by running the UNMODIFIED reference's SPIL
(GOPS @ /root/reference) on pyth_mobilerobot, on CPU.

TEST INFRASTRUCTURE.  Run in the build container only (`python oracle/make_golden_spil_robot.py`); it writes no other
file.  The reference draws the obstacle noise from NumPy's global RNG inside PythMobilerobotModel.forward; this script
wraps np.random.normal (the reference is untouched) to record every obstacle draw, as float32, in the order the passes
consume them.  Obstacle draws come in (v, w) pairs per forward call; the ego's std-0 draws are zeros and not stored.

spil_robot.npz: SPIL.local_update (spil.py:126-270), DetermPolicy / StateValue [64, 64] relu, action limits
+-[0.4, pi/3], forward_step 25, the shipped config's learning rates, four consecutive updates on one B = 128 batch of
reset-law states with crafted rows (obstacles that hit the robot, robots that leave x >= -2 or |y| <= 4, headings that
run past the 2 pi ClipObservation bound) and every seventh sample done.  Stored per update: the noise of both passes
[2][25][B][2], the tb values, the gradients, the post-update state_dict, safe_prob / lam / delta_i.

ckpt_spil_robot.npz: the shipped checkpoint results/SPIL/mobilerobot/apprfunc/apprfunc_16500_opt.pkl (its sha256 and its
tensors) and two known answers from it: a 30-step closed loop of the trained policy through the reference's wrapped
model from 32 reset-law states with recorded noise (observations, actions, rewards, constraints, dones), and one SPIL
update from the trained weights on a B = 256 batch (noise, tb values, gradients, safe_prob / lam / delta_i).

Discrete events are where fp32 round-off could move a result: the script refuses to write a file in which a constraint
value lies within 1e-4 of 0 (safe flag) or of 0.15 (crash), or a robot position within 1e-4 of x = -2 or |y| = 4."""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle.make_golden import OUT, _np, _sd, base_kwargs  # noqa: E402

H, B, N_UPDATES, B_CKPT, N_LOOP, K_LOOP = 25, 128, 4, 256, 32, 30
MARGIN = 1e-4
ACT_HI = np.array([0.4, np.pi / 3], dtype=np.float32)
CKPT = os.path.join("results", "SPIL", "mobilerobot", "apprfunc", "apprfunc_16500_opt.pkl")


def kwargs():
    return base_kwargs("pyth_mobilerobot", "SPIL", 13, 2, (64, 64), "relu", "DetermPolicy", forward_step=H,
                       constraint_dim=1, gamma=0.99, tau=0.005, action_high_limit=ACT_HI, action_low_limit=-ACT_HI,
                       value_learning_rate=2e-3, policy_learning_rate=3e-4)


def reset_states(n, seed, crafted=True):
    """The data env's reset box (env_ocp/pyth_mobilerobot.py:31-53) with the tracking error of its `reset`."""
    rs = np.random.RandomState(seed)
    lo = np.array([0, -1, -0.6, 0, 0, 0, 0, 0, 3.5, -3, np.pi / 2 - 0.3, 0, 0], dtype=np.float32)
    hi = np.array([2.7, 1, 0.6, 0.3, 0, 0, 0, 0, 6, 3, np.pi / 2 + 0.3, 0.5, 0], dtype=np.float32)
    o = (lo + rs.uniform(size=(n, 13)).astype(np.float32) * (hi - lo)).astype(np.float32)
    if crafted:
        o[0:8, 8], o[0:8, 9], o[0:8, 10], o[0:8, 11] = o[0:8, 0] + 1.0, o[0:8, 1], np.pi, 0.4   # head-on obstacle
        o[8:12, 0], o[8:12, 2], o[8:12, 3] = -1.999, np.pi, 0.4                                # leaves x >= -2
        o[12:16, 1], o[12:16, 2], o[12:16, 3] = 3.999, np.pi / 2, 0.4                          # leaves |y| <= 4
        o[16:20, 2], o[16:20, 4] = 6.28, 1.5                                                    # theta past 2 pi
    o[:, 5], o[:, 6], o[:, 7] = o[:, 1], o[:, 2], o[:, 3] - np.float32(0.3)
    return torch.from_numpy(o)


class Recorder:
    """np.random.normal in place of NumPy's: the same draws, rounded to float32 (what torch.Tensor makes of them
    anyway), with the obstacle's recorded."""

    def __init__(self):
        self.draws, self.real = [], np.random.normal

    def __enter__(self):
        def normal(loc=0.0, scale=1.0, size=None):
            v = self.real(loc, scale, size)
            if scale != 0:
                v = v.astype(np.float32)
                self.draws.append(v)
                v = v.astype(np.float64)
            return v
        np.random.normal = normal
        return self

    def __exit__(self, *exc):
        np.random.normal = self.real

    def take(self):
        """[calls][n][2] of the draws so far, then cleared."""
        d = np.stack([np.stack(self.draws[i:i + 2], -1) for i in range(0, len(self.draws), 2)])
        self.draws = []
        return d


def margin(c, nobs, done_in):
    """Distance of this step to its discrete events: the safe flag (c <= 0, every sample) and, for the samples still
    live, the crash (c > 0.15) and the bounds x < -2, |y| > 4 (a frozen sample's done flag is already set)."""
    live = ~done_in.bool()
    m = c.abs().min().item()
    if bool(live.any()):
        m = min(m, (c[live] - 0.15).abs().min().item(), (nobs[live, 0] + 2).abs().min().item(),
                (nobs[live, 1].abs() - 4).abs().min().item())
    return m


def watch(alg, seen):
    """Record the margins of every discrete event the reference's rollouts see (instrumentation of this script)."""
    fwd = alg.envmodel.forward

    def forward(o, a, d, info):
        out = fwd(o, a, d, info)
        seen.append(margin(out[3]["constraint"].detach(), out[0].detach(), d))
        return out
    alg.envmodel.forward = forward


def ref_batch(obs, done):
    n = obs.shape[0]
    return {"obs": obs.clone(), "done": done.clone(), "act": torch.zeros(n, 2), "rew": torch.zeros(n),
            "obs2": obs.clone(), "constraint": torch.zeros(n, 1)}


def record_update(alg, rec, prefix, obs, done, recorder, it):
    tb = alg.local_update(ref_batch(obs, done), it)
    noise = recorder.take()
    assert noise.shape == (2 * H, obs.shape[0], 2), noise.shape
    rec[prefix + "noise"] = noise.reshape(2, H, obs.shape[0], 2)
    for k, v in tb.items():
        if "Time" not in k:
            rec[f"{prefix}tb/{k}"] = np.float64(v)
    for nm in ("policy", "v"):
        for pn, p in getattr(alg.networks, nm).named_parameters():
            rec[f"{prefix}grad/{nm}.{pn}"] = _np(p.grad).copy()
    rec[prefix + "safe_prob"] = np.asarray(alg.safe_prob, dtype=np.float32)
    rec[prefix + "lam"] = np.asarray(alg.lam, dtype=np.float64)
    rec[prefix + "delta_i"] = np.asarray(alg.delta_i, dtype=np.float64)


def run_updates():
    from gops.create_pkg.create_alg import create_alg
    torch.manual_seed(4321)
    np.random.seed(4321)
    alg = create_alg(**kwargs())
    obs = reset_states(B, seed=92)
    done = torch.zeros(B)
    done[::7] = 1.0
    rec = {"in_obs": _np(obs), "in_done": _np(done)}
    for k, v in _sd(alg).items():
        rec["init/" + k] = v
    seen = []
    watch(alg, seen)
    with Recorder() as r:
        for it in range(N_UPDATES):
            record_update(alg, rec, f"it{it}/", obs, done, r, it)
            for k, v in _sd(alg).items():
                rec[f"it{it}/post/{k}"] = v
    assert min(seen) >= MARGIN, f"a discrete event lies within {MARGIN} ({min(seen):.3g})"
    print("updates: min margin", min(seen), {k: rec[k].tolist() for k in rec if k.endswith(("safe_prob", "lam"))})
    return rec


def run_checkpoint():
    from gops.create_pkg.create_alg import create_alg
    path = os.path.join(ref_shim.REFERENCE_ROOT, CKPT)
    with open(path, "rb") as f:
        sha = hashlib.sha256(f.read()).hexdigest()
    sd = torch.load(path, map_location="cpu", weights_only=False)
    rec = {"sha256": np.array(sha)}
    for k, v in sd.items():
        rec["ckpt/" + k] = _np(v).copy()
    torch.manual_seed(4322)
    np.random.seed(4322)
    alg = create_alg(**kwargs())
    alg.load_state_dict(sd)
    seen = []
    # closed loop of the trained policy (the evaluator's deterministic action) through the wrapped reference model
    obs = reset_states(N_LOOP, seed=93, crafted=False)
    done = torch.zeros(N_LOOP)
    rec["loop/obs0"] = _np(obs)
    traj = {"obs": [], "act": [], "rew": [], "con": [], "done": []}
    with Recorder() as r, torch.no_grad():
        for _ in range(K_LOOP):
            act = alg.networks.policy(obs)
            done_in = done
            obs, rew, d, info = alg.envmodel.forward(obs, act, done, {})
            c = info["constraint"]
            seen.append(margin(c, obs, done_in))
            done = d.float()
            for k, v in zip(traj, (obs, act, rew, c, done)):
                traj[k].append(_np(v).copy())
        rec["loop/noise"] = r.take()
    for k, v in traj.items():
        rec["loop/" + k] = np.stack(v)
    # one update from the trained weights
    watch(alg, seen)
    obs = reset_states(B_CKPT, seed=94)
    done = torch.zeros(B_CKPT)
    done[::5] = 1.0
    rec["upd/in_obs"], rec["upd/in_done"] = _np(obs), _np(done)
    with Recorder() as r:
        record_update(alg, rec, "upd/", obs, done, r, 0)
    assert min(seen) >= MARGIN, f"checkpoint: a discrete event lies within {MARGIN} ({min(seen):.3g})"
    print("checkpoint: min margin", min(seen), "dones", int(traj["done"][-1].sum()), "safe_prob", rec["upd/safe_prob"])
    return rec


if __name__ == "__main__":
    ref_shim.install()
    torch.set_num_threads(4)
    rec_u, rec_c = run_updates(), run_checkpoint()
    if "--dry" not in sys.argv:
        np.savez_compressed(os.path.join(OUT, "spil_robot.npz"), **rec_u)
        np.savez_compressed(os.path.join(OUT, "ckpt_spil_robot.npz"), **rec_c)
