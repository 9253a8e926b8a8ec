"""RPI (gops/algorithm/rpi.py) on pyth_oscillatorconti restated in PyTorch, in float32 or float64, replaying recorded
reset draws.  The Hamiltonian's parameter gradient comes from autograd's double backward (dV/dx with create_graph, then
backward through it), so it is independent of the hand derivation in csrc/rpi.cu.

TEST INFRASTRUCTURE: imported by tests only."""
import math

import numpy as np
import torch

ACTS = {"relu": torch.relu, "elu": torch.nn.functional.elu, "gelu": torch.nn.functional.gelu,
        "selu": torch.selu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}
KEYS = ("v.0.weight", "v.0.bias", "v.2.weight", "v.2.bias", "v.4.weight", "v.4.bias")


class Value:
    """StateValue [2 -> 64 -> 64 -> 1] as six leaf tensors."""

    def __init__(self, sd, act, dtype):
        self.p = [torch.as_tensor(np.asarray(sd[k]), dtype=dtype).clone().requires_grad_(True) for k in KEYS]
        self.act = ACTS[act]

    def __call__(self, x):
        w1, b1, w2, b2, w3, b3 = self.p
        h = self.act(x @ w1.T + b1)
        h = self.act(h @ w2.T + b2)
        return (h @ w3.T + b3).squeeze(-1)

    def grad_x(self, x, create_graph=False):
        x = x.detach().requires_grad_(True)
        (g,) = torch.autograd.grad(self(x).sum(), x, create_graph=create_graph)
        return g

    def flat(self):
        return torch.cat([t.detach().reshape(-1) for t in self.p])

    def state(self):
        return {k: t.detach().clone() for k, t in zip(KEYS, self.p)}


def action_and_adversary(target: Value, x, gamma_atte):
    p = target.grad_x(x).detach()
    a = -0.5 * (x[:, 0] * p[:, 1])
    w = 0.5 / gamma_atte ** 2 * (x[:, 1] * p[:, 1])
    return torch.stack([a, w], 1)


def wrapped_model(x, aw, gamma_atte):
    """delta_state and cost of the wrapped forward: ScaleAction [-1, 1] -> bounds, clipped (create_env_model chain)."""
    lo = torch.tensor([-5.0, -1.0 / gamma_atte], dtype=x.dtype)
    hi = -lo
    a = torch.clip(aw, -1.0, 1.0)
    a = torch.clip(lo + (hi - lo) * ((a + 1.0) / 2.0), lo, hi)
    return osc_f(x, a[:, 0], a[:, 1], gamma_atte)


def osc_f(x, u, w, gamma_atte):
    x0, x1 = x[:, 0], x[:, 1]
    d1 = 0.5 * (x0 ** 2 * x1) - 1 / (2 * gamma_atte ** 2) * x1 ** 3 - 0.5 * x1 + x0 * u + x1 * w
    f = torch.stack([-0.25 * x0, d1], 1)
    c = x0 ** 2 + x1 ** 2 + u ** 2 - gamma_atte ** 2 * w ** 2
    return f, c


def hamiltonian(value: Value, x, aw, gamma_atte, create_graph):
    f, c = wrapped_model(x, aw, gamma_atte)
    p = value.grad_x(x, create_graph=create_graph)
    return c + (p * f).sum(1)


def loss_and_grad(value: Value, x, aw, gamma_atte):
    """mean|H| and d/dparams by double backward (sign(0) = 0, as torch's abs)."""
    for t in value.p:
        t.grad = None
    loss = hamiltonian(value, x, aw, gamma_atte, True).abs().mean()
    loss.backward()
    # dV/dx does not depend on the output bias: its gradient stays None (Adam then skips it, as in the reference)
    return loss.detach(), torch.cat([(t.grad if t.grad is not None else torch.zeros_like(t)).reshape(-1)
                                     for t in value.p])


class Adam:
    """torch.optim.Adam(lr, betas=(0.9, 0.99)) over the value's leaves, state carried across Newton iterations."""

    def __init__(self, value: Value, lr=1e-3, betas=(0.9, 0.99), eps=1e-8):
        self.opt = torch.optim.Adam(value.p, lr=lr, betas=betas, eps=eps)


def run(sd0, act, gamma_atte, obs0, max_step, draws, n_iter, threshold=(5.0, 5.0), dt=1 / 200, lr=1e-3,
        max_steps=10000, dtype=torch.float64, counter0=0):
    """RPI.local_update x n_iter.  draws: list of [1 + n_k][B][2] per iteration (row 0 set_state).  Returns per
    iteration n, loss trace, H_after trace, H_before, and the final value state dict and Adam state."""
    value = Value(sd0, act, dtype)
    target = Value(sd0, act, dtype)
    opt = Adam(value, lr)
    x = torch.as_tensor(np.asarray(obs0), dtype=dtype).clone()
    cap = torch.as_tensor(np.asarray(max_step), dtype=torch.float64)
    cnt = counter0
    out = []
    for it in range(n_iter):
        d = torch.as_tensor(np.asarray(draws[it]), dtype=dtype)
        sx = d[0]
        saw = action_and_adversary(target, sx, gamma_atte)
        hb = hamiltonian(value, sx, saw, gamma_atte, False).abs().mean().item()
        losses, has = [], []
        n = 0
        while True:
            n += 1
            if n >= d.shape[0]:
                raise ValueError("draws exhausted")
            aw = action_and_adversary(target, x, gamma_atte)
            f, _ = osc_f(x, aw[:, 0], aw[:, 1], gamma_atte)
            xn = x + f * dt
            done = (xn[:, 0].abs() > threshold[0]) | (xn[:, 1].abs() > threshold[1])
            cnt += 1
            trunc = cnt > cap
            opt.opt.zero_grad()
            loss, _ = loss_and_grad(value, x, aw, gamma_atte)
            opt.opt.step()
            x = torch.where((done | trunc)[:, None], d[n], xn)
            ha = hamiltonian(value, sx, saw, gamma_atte, False).abs().mean().item()
            losses.append(loss.item())
            has.append(ha)
            if not (abs(ha) > 0.88 * abs(hb) and n < max_steps):
                break
        target = Value(value.state(), act, dtype)
        out.append(dict(n=n, loss=np.array(losses), h_after=np.array(has), h_before=hb, flat=value.flat().numpy().copy()))
    st = opt.opt.state
    mom = lambda t, k: st[t][k].reshape(-1) if k in st[t] else torch.zeros(t.numel(), dtype=dtype)
    adam = (torch.cat([mom(t, "exp_avg") for t in value.p]).numpy(),
            torch.cat([mom(t, "exp_avg_sq") for t in value.p]).numpy())
    return out, value.state(), adam, x.numpy(), cnt


def activation_derivs(act, z):
    """sigma', sigma'' in float64 NumPy (the hand formulas csrc/rpi.cu uses)."""
    z = np.asarray(z, dtype=np.float64)
    if act == "relu":
        return (z > 0).astype(np.float64), np.zeros_like(z)
    if act == "elu":
        e = np.exp(z)
        return np.where(z > 0, 1.0, e), np.where(z > 0, 0.0, e)
    if act == "selu":
        sc, al = 1.0507009873554805, 1.6732632423543772
        e = np.exp(z)
        return np.where(z > 0, sc, sc * al * e), np.where(z > 0, 0.0, sc * al * e)
    if act == "gelu":
        phi = np.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
        from scipy.special import erf
        cdf = 0.5 * (1 + erf(z / math.sqrt(2)))
        return cdf + z * phi, phi * (2 - z * z)
    if act == "sigmoid":
        s = 1 / (1 + np.exp(-z))
        d = s * (1 - s)
        return d, d * (1 - 2 * s)
    if act == "tanh":
        t = np.tanh(z)
        d = 1 - t * t
        return d, -2 * t * d
    raise ValueError(act)


def hand_loss_grad(sd, act, x, f, c):
    """mean|c + V'| and its parameter gradient by the forward-tangent / reverse formulas of csrc/rpi.cu, float64 NumPy."""
    act_f = {"relu": lambda z: np.maximum(z, 0), "elu": lambda z: np.where(z > 0, z, np.expm1(z)),
             "selu": lambda z: 1.0507009873554805 * np.where(z > 0, z, 1.6732632423543772 * np.expm1(z)),
             "sigmoid": lambda z: 1 / (1 + np.exp(-z)), "tanh": np.tanh,
             "gelu": lambda z: z * 0.5 * (1 + __import__("scipy.special", fromlist=["erf"]).erf(z / math.sqrt(2)))}[act]
    W1, b1, W2, b2, W3, b3 = [np.asarray(sd[k], dtype=np.float64) for k in KEYS]
    B = x.shape[0]
    z1 = x @ W1.T + b1
    h1 = act_f(z1)
    d1, s1 = activation_derivs(act, z1)
    zt1 = f @ W1.T
    ht1 = d1 * zt1
    z2 = h1 @ W2.T + b2
    zt2 = ht1 @ W2.T
    d2, s2 = activation_derivs(act, z2)
    ht2 = d2 * zt2
    vd = ht2 @ W3[0]
    H = c + vd
    q = np.sign(H) / B
    gzt2 = q[:, None] * W3[0] * d2
    gz2 = q[:, None] * W3[0] * zt2 * s2
    gW3 = (q[:, None] * ht2).sum(0)[None]
    gW2 = gzt2.T @ ht1 + gz2.T @ h1
    gb2 = gz2.sum(0)
    ght1 = gzt2 @ W2
    gh1 = gz2 @ W2
    gzt1 = ght1 * d1
    gz1 = gh1 * d1 + ght1 * zt1 * s1
    gW1 = gzt1.T @ f + gz1.T @ x
    gb1 = gz1.sum(0)
    grad = np.concatenate([gW1.ravel(), gb1, gW2.ravel(), gb2, gW3.ravel(), np.zeros(1)])
    return np.abs(H).mean(), grad
