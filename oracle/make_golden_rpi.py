"""Generate tests/golden/rpi_osc_{a,b,c}.npz by running the UNMODIFIED reference's RPI (the GOPS tree that
oracle/ref_shim.py finds) on pyth_oscillatorconti with the settings of
example_train/rpi/rpi_mlp_oscillatorconti_onserial.py, on CPU.

TEST INFRASTRUCTURE.  Run where the reference is available (`python oracle/make_golden_rpi.py`); it writes no other
file.  The reference draws its reset states and episode caps from NumPy's global RNG (pyth_oscillatorconti_model.py max_step /
reset); this script wraps np.random.uniform (the reference is untouched) to record every draw, as float32 for states
(what `.float()` makes of them) and as float64 for the caps (the raw U[lower_step, upper_step) draws, before the floor).

  (a) the shipped config, B = 64, 13 Newton iterations (past the step at which the first samples are truncated);
  (b) B = 256, lower_step / upper_step 5 / 40 and initial_state_range [4.5, 4.5], so that done samples, truncation and
      action clipping all occur (asserted);
  (c) the shipped config with max_step_update_value = 3.

Stored: the initial value weights, the first reset and the episode caps, the draws of every Newton iteration once
([sum_k (1 + n_k)][B][2], offsets per iteration), per iteration n, the loss and H_after traces, H_before and the value
weights at its end, and the final Adam state.  Discrete events are where float round-off could change a result: the
script refuses to write a case in which a stopping ratio H_after / (0.88 H_before) lies within 1e-4 of 1, a sampled
|x_i'| within 1e-4 of its threshold, or a Hamiltonian |H_i| of the loss within 1e-4 of 0; it then tries the next seed."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
MARGIN = 1e-4
KEYS = ("v.0.weight", "v.0.bias", "v.2.weight", "v.2.bias", "v.4.weight", "v.4.bias")


def kwargs(B=64, lower=100, upper=200, rng=(1.2, 1.2), max_step_update_value=10000, seed=0):
    return dict(env_id="pyth_oscillatorconti", algorithm="RPI", enable_cuda=False, use_gpu=False, is_adversary=True,
                is_constrained=False, is_render=False, value_func_name="StateValue", value_func_type="MLP",
                value_hidden_sizes=[64, 64], value_hidden_activation="elu", value_output_activation="linear",
                policy_func_name="DetermPolicy", policy_func_type="POLY", policy_act_distribution="default",
                learning_rate=1e-3, gamma_atte=2.0, trainer="on_serial_trainer", max_newton_iteration=50,
                max_step_update_value=max_step_update_value, max_iteration=50, sample_batch_size=B,
                reset_batch_size=B, fixed_initial_state=[0.5, -0.5], initial_state_range=list(rng),
                state_threshold=[5.0, 5.0], lower_step=lower, upper_step=upper, max_episode_steps=200, seed=seed,
                obsv_dim=2, action_dim=1, action_type="continu", cnn_shared=False,
                action_high_limit=np.ones(1, np.float32), action_low_limit=-np.ones(1, np.float32))


class Recorder:
    def __init__(self):
        self.draws, self.real = [], np.random.uniform

    def __enter__(self):
        def uniform(low=0.0, high=1.0, size=None):
            v = self.real(low, high, size)
            self.draws.append(np.asarray(v))
            return v
        np.random.uniform = uniform
        return self

    def __exit__(self, *exc):
        np.random.uniform = self.real

    def take_resets(self):
        """[calls][B][2] float32 of the reset() calls recorded so far (two uniform draws of [B, 1] each), then cleared."""
        d = self.draws
        assert len(d) % 2 == 0
        out = np.stack([np.concatenate([d[i], d[i + 1]], 1) for i in range(0, len(d), 2)]).astype(np.float32)
        self.draws = []
        return out


def run_case(n_iter, seed, **kw):
    ref_shim.install()
    from gops.create_pkg.create_alg import create_alg
    torch.manual_seed(seed)
    np.random.seed(seed)
    rec = {}
    margins = {"ratio": [], "thr": [], "H": []}
    events = {"done": 0, "trunc": 0, "clip": 0}
    with Recorder() as r:
        alg = create_alg(**kwargs(seed=seed, **kw))
        d = r.draws
        rec["max_step"] = np.asarray(d[0], dtype=np.float64)
        rec["obs0"] = np.concatenate([d[1], d[2]], 1).astype(np.float32)
        r.draws = []
        sd = alg.networks.state_dict()
        for k in KEYS:
            rec["init/" + k] = sd["value." + k].numpy().copy()
        th = np.array(alg.env_model.state_threshold)
        hs = []
        calc = alg._RPI__calculate_norm_hamiltonian
        alg._RPI__calculate_norm_hamiltonian = lambda s: hs.append(calc(s)) or hs[-1]
        losses = []
        comp = alg._RPI__compute_loss

        def compute_loss(data):
            obs, aw = data["obs"], torch.cat((data["act"], data["advers"]), 1)
            events["clip"] += int((aw.abs() > 1).any())
            # the per-sample Hamiltonian of this loss (reference code path, recomputed for the margin)
            o = obs.clone().requires_grad_(True)
            (dv,) = torch.autograd.grad(alg.networks.value(o).sum(), o)
            _, rew, _, info = alg.env_model.forward(obs, aw, torch.zeros(obs.shape[0]).bool(), {})
            margins["H"].append(float((-rew + (dv * info["delta_state"]).sum(1)).abs().min()))
            nx = data["obs2"]
            margins["thr"].append(float(np.abs(np.abs(nx.numpy()) - th).min()))
            events["done"] += int(data["done"].sum())
            events["trunc"] += int(data["time_limited"].sum())
            loss = comp(data)
            losses.append(loss.item())
            return loss
        alg._RPI__compute_loss = compute_loss
        offs, draws = [0], []
        for it in range(n_iter):
            hs.clear()
            losses.clear()
            alg.local_update(None, it)
            n = alg.num_update_value
            dr = r.take_resets()
            assert dr.shape[0] == 1 + n, (dr.shape, n)
            draws.append(dr)
            offs.append(offs[-1] + dr.shape[0])
            rec[f"it{it}/n"] = np.int64(n)
            rec[f"it{it}/h_before"] = np.float64(hs[0])
            rec[f"it{it}/h_after"] = np.array(hs[1:], dtype=np.float64)
            rec[f"it{it}/loss"] = np.array(losses, dtype=np.float64)
            margins["ratio"] += [abs(h / (0.88 * hs[0]) - 1) for h in hs[1:]]
            sd = alg.networks.state_dict()
            rec[f"it{it}/flat"] = np.concatenate([sd["value." + k].numpy().reshape(-1) for k in KEYS])
        rec["draws"] = np.concatenate(draws)
        rec["draw_offsets"] = np.array(offs, dtype=np.int64)
        st = alg.approximate_optimizer.state
        ps = list(alg.networks.value.parameters())
        # the output bias never gets a gradient (dV/dx does not depend on it), so Adam keeps no state for it
        mom = lambda p, k: st[p][k].numpy().reshape(-1) if k in st[p] else np.zeros(p.numel(), np.float32)
        rec["adam/exp_avg"] = np.concatenate([mom(p, "exp_avg") for p in ps])
        rec["adam/exp_avg_sq"] = np.concatenate([mom(p, "exp_avg_sq") for p in ps])
        rec["adam/step"] = np.int64(int(st[ps[0]]["step"]))
        rec["final_obs"] = alg.obs.numpy().copy()
    m = {k: (min(v) if v else 1.0) for k, v in margins.items()}
    return rec, m, events


def main():
    cases = {"a": (13, dict()), "b": (6, dict(B=256, lower=5, upper=40, rng=(4.5, 4.5))),
             "c": (6, dict(max_step_update_value=3))}
    only = sys.argv[1:] or list(cases)
    for name in only:
        n_iter, kw = cases[name]
        for seed in range(0, 50):
            rec, m, ev = run_case(n_iter, seed, **kw)
            ok = all(v > MARGIN for v in m.values())
            if name == "b":
                ok = ok and all(v > 0 for v in ev.values())
            print(name, "seed", seed, "n", [int(rec[f"it{i}/n"]) for i in range(n_iter)], "margins", m, "events", ev)
            if ok:
                rec["seed"] = np.int64(seed)
                rec["config"] = np.array(repr(kw))
                np.savez_compressed(os.path.join(OUT, f"rpi_osc_{name}.npz"), **rec)
                break
        else:
            raise SystemExit(f"case {name}: no seed without a discrete event within {MARGIN} of flipping")


if __name__ == "__main__":
    main()
