"""CPU oracle of SPIL (gops/algorithm/spil.py) -- TEST INFRASTRUCTURE, not the product.

A restatement in PyTorch (fp32 or fp64) and NumPy of the reference's two loss passes and its PI multiplier controller,
built on the env models and nets of oracle/gops_oracle.py:

  spil_loss_value   __compute_loss_v       spil.py:182-212
  spil_loss_policy  __compute_loss_policy  spil.py:214-255 (Phi :224-232)
  spil_weights      __spil_get_weight      spil.py:257-270

Golden vectors of the unmodified reference: oracle/make_golden_spil.py -> tests/golden/spil_*.npz."""
from typing import Dict, Tuple

import numpy as np
import torch

KP, KI, KD, CHANCE_THRE = 60, 0.02, 0, 0.97     # spil.py:106-112


def phi(y: torch.Tensor) -> torch.Tensor:
    """Constraint -> cost transform, spil.py:224-232: m1 = 1, m2 = m1 / (1 + m1) * 0.9, tau = 0.07 (python scalars)."""
    m1, tau = 1, 0.07
    m2 = m1 / (1 + m1) * 0.9
    return (1 + tau * m1) / (1 + m2 * tau * torch.exp(torch.clamp(y / tau, min=-10, max=5)))


def spil_loss_value(v, policy, v_target, env, data: dict, forward_step: int, gamma: float):
    """(loss_v, mean v(o), traj_issafe [B, 2]).  The backup's terminal value is NOT masked by done, and a trajectory is
    safe for constraint i when info["constraint"][:, i] <= 0 on every step."""
    o, d, info = data["obs"], data["done"], data
    val = v.value(o)
    with torch.no_grad():
        issafe = torch.ones(o.shape[0], 2, dtype=o.dtype)
        backup = None
        for step in range(forward_step):
            a = policy.act(o)
            o, r, d, info = env.forward(o, a, d, info)
            backup = r if step == 0 else backup + gamma ** step * r
            issafe = issafe * (info["constraint"] <= 0)
        backup = backup + gamma ** forward_step * v_target.value(o)
    return ((val - backup) ** 2).mean(), val.mean(), issafe


def safe_probability(issafe: torch.Tensor) -> np.ndarray:
    """traj_issafe.mean(0) of the reference: a float32 mean."""
    return issafe.float().mean(0).numpy()


def spil_loss_policy(policy, env, data: dict, forward_step: int, gamma: float, w_r: float, w_c) -> torch.Tensor:
    """-mean(w_r sum_k gamma^k r_k + sum_i w_c,i prod_k Phi(c_k,i)); w_c is applied as a float32 (or oracle-dtype)
    tensor, w_r as a python float, as the reference does."""
    o, d, info = data["obs"], data["done"], data
    ret = prod = None
    for step in range(forward_step):
        a = policy.act(o)
        o, r, d, info = env.forward(o, a, d, info)
        c = phi(info["constraint"])
        ret = r if step == 0 else ret + gamma ** step * r
        prod = c if step == 0 else prod * c
    wc = torch.tensor(np.asarray(w_c, dtype=np.float64), dtype=o.dtype)
    return -(float(w_r) * ret + (prod * wc).sum(1)).mean()


def new_controller(n: int = 2) -> Dict[str, np.ndarray]:
    """Controller state at construction (spil.py:106-112)."""
    return {"delta_i": np.zeros(n), "safe_prob_pre": np.zeros(n), "lam": np.zeros(n)}


def spil_weights(state: Dict[str, np.ndarray], safe_prob: np.ndarray, Kp=KP, Ki=KI, Kd=KD,
                 chance_thre=None) -> Tuple[float, np.ndarray]:
    """One controller step on `state` (updated in place); returns (w_r, w_c) in float64.  NumPy dtype rules are kept:
    safe_prob is float32, so from the second step on safe_prob_pre - safe_prob is a float32 difference and Kd * delta_d
    a float32 product."""
    thre = np.array([CHANCE_THRE] * len(safe_prob)) if chance_thre is None else np.asarray(chance_thre)
    dp = thre - safe_prob
    big = np.abs(dp)
    sep = np.where(big > 0.1, dp * 0.7, dp)
    sep = np.where(big > 0.2, dp * 0, sep)
    state["delta_i"] = np.clip(state["delta_i"] + sep, 0, 99999)
    dd = np.clip(state["safe_prob_pre"] - safe_prob, 0, 3333)
    lam = np.clip(Ki * state["delta_i"] + Kp * dp + Kd * dd, 0, 3333)
    state["safe_prob_pre"] = safe_prob
    state["lam"] = lam
    total = 1 + lam.sum()
    return 1 / total, lam / total
