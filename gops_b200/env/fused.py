"""Bridge between the (descriptor-style) env-model / wrapper objects and the fused CUDA kernels.

`collect_chain(top)` walks a wrapper chain assembled by `create_env_model` and returns the
constants the kernels need; `fill_plan_desc` writes them into the C struct; `fused_forward`
implements `envmodel.forward(obs, action, done, info)` for any level of the chain with one
`gops_b200_model_step` launch.
"""
import ctypes as C

import numpy as np
import torch

from gops_b200 import _lib


def collect_chain(top) -> dict:
    cfg = dict(action_scale=0, clip_action=0, clip_obs=0, mask_at_done=0, reward_shaping=0,
               reward_shift=0.0, reward_scale=1.0, min_action=None, max_action=None,
               obs_scaling=0, obs_scale=None, obs_shift=None, repeat_num=0, sum_reward=1)
    m = top
    while hasattr(m, "model"):
        m.describe(cfg)
        m = m.model
    cfg["base"] = m
    return cfg


def _fill(arr, values, n):
    vals = np.asarray(values, dtype=np.float32).reshape(-1)
    for i in range(n):
        arr[i] = float(vals[i]) if i < len(vals) else 0.0


def fill_plan_desc(desc: _lib.PlanDesc, top, policy_low, policy_high):
    cfg = collect_chain(top)
    base = cfg["base"]
    na = base.action_dim
    if na > _lib.MAX_ACT:
        raise NotImplementedError(f"action_dim {na} > {_lib.MAX_ACT} not supported by the fused kernels")
    for k in ("action_scale", "clip_action", "clip_obs", "mask_at_done", "reward_shaping"):
        setattr(desc, k, int(cfg[k]))
    desc.reward_shift, desc.reward_scale = float(cfg["reward_shift"]), float(cfg["reward_scale"])
    lo = base.action_lower_bound.detach().cpu().numpy()
    hi = base.action_upper_bound.detach().cpu().numpy()
    _fill(desc.act_low, lo, na)
    _fill(desc.act_high, hi, na)
    _fill(desc.min_action, cfg["min_action"] if cfg["min_action"] is not None else -np.ones(na), na)
    _fill(desc.max_action, cfg["max_action"] if cfg["max_action"] is not None else np.ones(na), na)
    _fill(desc.pol_act_low, policy_low if policy_low is not None else -np.ones(na), na)
    _fill(desc.pol_act_high, policy_high if policy_high is not None else np.ones(na), na)
    desc.repeat_num, desc.sum_reward = int(cfg["repeat_num"]), int(cfg["sum_reward"])
    desc.obs_scaling = int(cfg["obs_scaling"])
    if cfg["obs_scaling"]:
        n = base.obs_dim
        sc = (C.c_float * n)(*[float(v) for v in cfg["obs_scale"]])
        sh = (C.c_float * n)(*[float(v) for v in cfg["obs_shift"]])
        desc.obs_scale, desc.obs_shift = C.cast(sc, C.POINTER(C.c_float)), C.cast(sh, C.POINTER(C.c_float))
        cfg["_keepalive"] = (sc, sh)      # the C side copies the arrays during plan_create
    base.fill_plan_desc(desc)
    return cfg


def _dummy_mlp(obs_dim, act_dim):
    return _lib.MlpDesc(obs_dim, 0, 64, act_dim, _lib.ACT_IDS["relu"], _lib.ACT_IDS["linear"])


class _StepPlan:
    def __init__(self, top, device):
        with torch.cuda.device(device):
            self._create(top)

    def _create(self, top):
        base = top.unwrapped
        desc = _lib.PlanDesc()
        desc.alg, desc.horizon, desc.gamma = _lib.ALG_FHADP, 1, 1.0
        desc.policy = _dummy_mlp(base.obs_dim, base.action_dim)
        keep = fill_plan_desc(desc, top, None, None)
        self.handle = C.c_void_p()
        _lib.check(_lib.lib().gops_b200_plan_create(C.byref(desc), C.byref(self.handle)))

    def __del__(self):
        try:
            if self.handle:
                _lib.lib().gops_b200_plan_destroy(self.handle)
        except Exception:
            pass


def make_batch(base, obs, done, info, keep):
    """Build the C batch struct; `keep` collects tensors that must stay alive until launch."""
    dev = obs.device
    f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
    b = _lib.Batch()
    o, d = f32(obs), f32(done)
    keep += [o, d]
    b.batch, b.obs, b.done = o.shape[0], o.data_ptr(), d.data_ptr()
    base.fill_batch(b, info, f32, keep)
    return b


def fused_forward(top, obs, action, done, info):
    if not torch.cuda.is_available():
        raise RuntimeError("gops_b200 env models run on a CUDA device only (no CPU fallback)")
    src = obs.device
    dev = obs.device if obs.is_cuda else torch.device("cuda", torch.cuda.current_device())
    plans = top.__dict__.setdefault("_step_plans", {})     # one per device
    plan = plans.get(dev.index)
    if plan is None:
        plan = plans[dev.index] = _StepPlan(top, dev)
    base = top.unwrapped
    keep = []
    obs_d = obs.detach().to(dev, torch.float32)
    with torch.cuda.device(dev):
        info_d = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in (info or {}).items()}
        b = make_batch(base, obs_d, done.to(dev), info_d, keep)
        act = action.detach().to(dev, torch.float32).contiguous()
        B = obs_d.shape[0]
        nobs = torch.empty((B, base.obs_dim), dtype=torch.float32, device=dev)
        rew = torch.empty(B, dtype=torch.float32, device=dev)
        ndone = torch.empty(B, dtype=torch.float32, device=dev)
        extra = base.alloc_next_info(B, dev)
        if hasattr(base, "model_io"):        # models with noise and constraints: this step's draws, the constraint out
            noise, extra["constraint"] = base.model_io(B, dev)
            keep.append(noise)
            _lib.check(_lib.lib().gops_b200_plan_set_model_io(plan.handle, _lib.ptr(noise), _lib.ptr(extra["constraint"])))
        _lib.check(_lib.lib().gops_b200_model_step(
            plan.handle, C.byref(b), _lib.ptr(act), _lib.ptr(nobs), _lib.ptr(rew), _lib.ptr(ndone),
            _lib.ptr(extra.get("state")), _lib.ptr(extra.get("ref_points")), _lib.ptr(extra.get("ref_time")),
            _lib.stream_ptr()))
        if hasattr(base, "model_io"):        # the buffers are this call's: a later call must set its own
            _lib.check(_lib.lib().gops_b200_plan_set_model_io(plan.handle, None, None))
    extra["_obs_in"] = obs_d if not getattr(top, "_scales_obs", False) else obs_d     # constraint providers read the incoming obs
    next_info = base.make_next_info(info, extra)
    return nobs.to(src), rew.to(src), (ndone != 0).to(src), next_info
