"""MLP approximate functions of the ADP hot path, H100 edition.

Same constructor kwargs, class names, `state_dict` keys and init as the reference
(gops/apprfunc/mlp.py: mlp() :36-41, DetermPolicy :50-77, FiniteHorizonPolicy :80-111,
ActionValue :224-245, StateValue :309-329); `forward` runs the fused sm_90a inference kernels
(`gops_b200_mlp_forward`) instead of nn.Sequential.  Training never calls `forward`: the
algorithms hand the flat parameter vector to the fused rollout kernel.
"""
__all__ = ["DetermPolicy", "FiniteHorizonPolicy", "FiniteHorizonFullPolicy", "StochaPolicy", "ActionValue", "ActionValueDistri",
           "StateValue"]

import ctypes as C

import numpy as np
import torch
import torch.nn as nn

from gops_b200 import _lib
from gops_b200.utils.act_distribution_cls import Action_Distribution
from gops_b200.utils.common_utils import activation_name, get_activation_func
from gops_b200.utils.flat_params import FlatParams


def mlp(sizes, activation, output_activation=nn.Identity):
    """nn.Sequential(Linear, act, ..., Linear, out_act): parameter container with torch default init."""
    layers = []
    for j in range(len(sizes) - 1):
        act = activation if j < len(sizes) - 2 else output_activation
        layers += [nn.Linear(sizes[j], sizes[j + 1]), act()]
    return nn.Sequential(*layers)


def count_vars(module):
    return sum([np.prod(p.shape) for p in module.parameters()])


class _FusedMlp(nn.Module, Action_Distribution):
    """Shared plumbing: shape checks, flat parameter view, ctypes descriptor, fused inference."""

    _net_attr = "pi"
    _time_input = False

    def _build(self, in_dim, out_dim, kwargs):
        hidden = list(kwargs["hidden_sizes"])
        if len(hidden) != 2 or hidden[0] != hidden[1]:
            raise NotImplementedError(
                f"gops_b200 fused MLP kernels need two equal hidden layers, got hidden_sizes={hidden}")
        if hidden[0] not in (64, 256):
            raise NotImplementedError(f"gops_b200 fused MLP kernels are built for hidden widths 64 and 256, got {hidden[0]}")
        self._obs_dim, self._out_dim, self._hidden = in_dim, out_dim, hidden[0]
        self._hidden_act = kwargs["hidden_activation"]
        self._out_act = kwargs.get("output_activation", "linear")
        if self._out_act != "linear":
            raise NotImplementedError("gops_b200 fused MLP kernels support output_activation='linear' only")
        net = mlp([in_dim + int(self._time_input)] + hidden + [out_dim],
                  get_activation_func(self._hidden_act), get_activation_func(self._out_act))
        setattr(self, self._net_attr, net)
        self.action_distribution_cls = kwargs["action_distribution_cls"]
        self.__dict__["_flat_params"] = FlatParams(getattr(self, self._net_attr))

    @property
    def flat_params(self) -> FlatParams:
        return self.__dict__["_flat_params"]

    def mlp_desc(self) -> _lib.MlpDesc:
        return _lib.MlpDesc(self._obs_dim, int(self._time_input), self._hidden, self._out_dim,
                            _lib.ACT_IDS[self._hidden_act], _lib.ACT_IDS[self._out_act])

    def _infer(self, obs: torch.Tensor, virtual_t: float, squash: bool) -> torch.Tensor:
        flat = self.flat_params.sync()
        if not flat.is_cuda:
            raise RuntimeError("gops_b200 apprfuncs run on a CUDA device only (no CPU fallback); call .cuda()")
        src_dev = obs.device
        x = obs.detach().to(flat.device, torch.float32)
        squeeze = x.dim() == 1
        x = x.reshape(-1, self._obs_dim).contiguous()
        out = torch.empty((x.shape[0], self._out_dim), dtype=torch.float32, device=flat.device)
        lo = hi = None
        if squash:
            lo = (C.c_float * self._out_dim)(*self.act_low_lim.detach().cpu().tolist())
            hi = (C.c_float * self._out_dim)(*self.act_high_lim.detach().cpu().tolist())
        desc = self.mlp_desc()
        with torch.cuda.device(flat.device):
            _lib.check(_lib.lib().gops_b200_mlp_forward(
                C.byref(desc), _lib.ptr(flat), _lib.ptr(x), x.shape[0], float(virtual_t), lo, hi,
                _lib.ptr(out), _lib.stream_ptr()))
        if squeeze:
            out = out[0]
        return out.to(src_dev)


class DetermPolicy(_FusedMlp):
    """Deterministic policy: obs -> action (reference mlp.py:50-77)."""

    def __init__(self, **kwargs):
        super().__init__()
        self._build(kwargs["obs_dim"], kwargs["act_dim"], kwargs)
        self.register_buffer("act_high_lim", torch.from_numpy(np.asarray(kwargs["act_high_lim"], dtype=np.float32)))
        self.register_buffer("act_low_lim", torch.from_numpy(np.asarray(kwargs["act_low_lim"], dtype=np.float32)))

    def forward(self, obs):
        return self._infer(obs, 0.0, squash=True)


class FiniteHorizonPolicy(_FusedMlp):
    """Finite-horizon deterministic policy: (obs, virtual_t) -> action (reference mlp.py:80-111)."""

    _time_input = True

    def __init__(self, **kwargs):
        super().__init__()
        self._build(kwargs["obs_dim"], kwargs["act_dim"], kwargs)
        self.register_buffer("act_high_lim", torch.from_numpy(np.asarray(kwargs["act_high_lim"], dtype=np.float32)))
        self.register_buffer("act_low_lim", torch.from_numpy(np.asarray(kwargs["act_low_lim"], dtype=np.float32)))

    def forward(self, obs, virtual_t=1):
        return self._infer(obs, float(virtual_t), squash=True)


class FiniteHorizonFullPolicy(nn.Module, Action_Distribution):
    """Open-loop finite-horizon policy (reference mlp.py:114-145): ONE evaluation on obs emits the actions of all
    `pre_horizon` steps; `forward` returns the first one.  Evaluated by the layer-wise wgmma MLP
    (gops_b200_mlpnet_*); trained by FHADP2 through the fused open-loop rollout."""

    def __init__(self, **kwargs):
        super().__init__()
        hidden = list(kwargs["hidden_sizes"])
        if len(hidden) != 2 or hidden[0] != hidden[1] or hidden[0] > 256:
            raise NotImplementedError(f"gops_b200 FiniteHorizonFullPolicy: two equal hidden layers <= 256, got {hidden}")
        self._obs_dim, self.act_dim, self.pre_horizon = kwargs["obs_dim"], kwargs["act_dim"], kwargs["pre_horizon"]
        if self.act_dim * self.pre_horizon > 256:
            raise NotImplementedError("gops_b200 FiniteHorizonFullPolicy: act_dim * pre_horizon must be <= 256")
        self._hidden, self._hidden_act = hidden[0], kwargs["hidden_activation"]
        if kwargs.get("output_activation", "linear") != "linear":
            raise NotImplementedError("gops_b200 fused MLP kernels support output_activation='linear' only")
        self.pi = mlp([self._obs_dim] + hidden + [self.act_dim * self.pre_horizon],
                      get_activation_func(self._hidden_act), get_activation_func("linear"))
        self.register_buffer("act_high_lim", torch.from_numpy(np.asarray(kwargs["act_high_lim"], dtype=np.float32)))
        self.register_buffer("act_low_lim", torch.from_numpy(np.asarray(kwargs["act_low_lim"], dtype=np.float32)))
        self.action_distribution_cls = kwargs["action_distribution_cls"]
        self.__dict__["_flat_params"] = FlatParams(self.pi)
        self.__dict__["_net"] = None

    @property
    def flat_params(self) -> FlatParams:
        return self.__dict__["_flat_params"]

    def mlp_desc(self) -> _lib.MlpDesc:
        return _lib.MlpDesc(self._obs_dim, 0, self._hidden, self.act_dim * self.pre_horizon,
                            _lib.ACT_IDS[self._hidden_act], _lib.ACT_IDS["linear"])

    def forward(self, obs):
        return self.forward_all_policy(obs)[:, 0, :]

    def forward_all_policy(self, obs):
        from gops_b200.ops.layerwise_mlp import LayerwiseMlp
        flat = self.flat_params.sync()
        if not flat.is_cuda:
            raise RuntimeError("gops_b200 apprfuncs run on a CUDA device only (no CPU fallback); call .cuda()")
        src = obs.device
        x = obs.detach().to(flat.device, torch.float32).reshape(-1, self._obs_dim).contiguous()
        net = self.__dict__["_net"]
        if net is None or net.max_batch < x.shape[0] or net.device != flat.device:
            net = self.__dict__["_net"] = LayerwiseMlp([self._obs_dim, self._hidden, self._hidden,
                                                        self.act_dim * self.pre_horizon], self._hidden_act,
                                                       max_batch=max(x.shape[0], 1024), device=flat.device)
        net.pack(flat)
        z = net.forward(x, train=False).reshape(x.shape[0], self.pre_horizon, self.act_dim)
        # the squashing below is 3 elementwise ops on [B, H, A] at inference time only (training fuses it)
        act = (self.act_high_lim - self.act_low_lim) / 2 * torch.tanh(z) + (self.act_high_lim + self.act_low_lim) / 2
        return act.to(src)


class _LayerwiseNet(nn.Module):
    """A general `mlp()` network (any depth, widths <= 256) evaluated by the layer-wise wgmma MLP."""

    _attr = "net"

    def _build_net(self, sizes, hidden_activation, output_activation="linear"):
        if output_activation != "linear":
            raise NotImplementedError("gops_b200 fused MLP kernels support output_activation='linear' only")
        if max(sizes) > 256 or len(sizes) > 9:
            raise NotImplementedError(f"gops_b200 layer-wise MLP: widths <= 256, <= 8 layers, got {sizes}")
        self._sizes, self._hidden_act = [int(v) for v in sizes], hidden_activation
        setattr(self, self._attr, mlp(self._sizes, get_activation_func(hidden_activation), get_activation_func("linear")))
        self.__dict__["_flat_params"] = FlatParams(getattr(self, self._attr))
        self.__dict__["_nets"] = {}

    @property
    def flat_params(self) -> FlatParams:
        return self.__dict__["_flat_params"]

    def layerwise(self, max_batch: int, slots: int = 1, tag: str = "infer"):
        """The library handle for this network (one per use: inference, training slots); created on first use."""
        from gops_b200.ops.layerwise_mlp import LayerwiseMlp
        flat = self.flat_params.sync()
        if not flat.is_cuda:
            raise RuntimeError("gops_b200 apprfuncs run on a CUDA device only (no CPU fallback); call .cuda()")
        net = self.__dict__["_nets"].get(tag)
        if net is None or net.max_batch < max_batch or net.slots < slots or net.device != flat.device:
            net = self.__dict__["_nets"][tag] = LayerwiseMlp(self._sizes, self._hidden_act, max_batch=max(max_batch, 256),
                                                             slots=slots, device=flat.device)
        return net

    def _raw(self, x: torch.Tensor) -> torch.Tensor:
        flat = self.flat_params.sync()
        net = self.layerwise(x.shape[0])
        net.pack(flat)
        return net.forward(x, train=False)


class StochaPolicy(_LayerwiseNet, Action_Distribution):
    """Stochastic policy: obs -> (mean, std) of the pre-squash Gaussian (reference mlp.py:149-221, std_type
    "mlp_shared": one network emits mean and log_std)."""

    _attr = "policy"

    def __init__(self, **kwargs):
        super().__init__()
        self.std_type = kwargs["std_type"]
        if self.std_type != "mlp_shared":
            raise NotImplementedError(f"gops_b200 StochaPolicy implements std_type='mlp_shared', got {self.std_type}")
        self._obs_dim, self.act_dim = kwargs["obs_dim"], kwargs["act_dim"]
        self._build_net([self._obs_dim] + list(kwargs["hidden_sizes"]) + [self.act_dim * 2], kwargs["hidden_activation"],
                        kwargs.get("output_activation", "linear"))
        self.min_log_std, self.max_log_std = kwargs["min_log_std"], kwargs["max_log_std"]
        self.register_buffer("act_high_lim", torch.from_numpy(np.asarray(kwargs["act_high_lim"], dtype=np.float32)))
        self.register_buffer("act_low_lim", torch.from_numpy(np.asarray(kwargs["act_low_lim"], dtype=np.float32)))
        self.action_distribution_cls = kwargs["action_distribution_cls"]

    def forward(self, obs):
        src = obs.device
        flat = self.flat_params.sync()
        x = obs.detach().to(flat.device, torch.float32).reshape(-1, self._obs_dim).contiguous()
        logits = self._raw(x)
        mean, log_std = torch.chunk(logits, chunks=2, dim=-1)
        std = torch.clamp(log_std, self.min_log_std, self.max_log_std).exp()       # 2 elementwise ops, inference only
        return torch.cat((mean, std), dim=-1).to(src)


class ActionValue(_LayerwiseNet, Action_Distribution):
    """Action value: (obs, act) -> q (reference mlp.py:224-245), the critic of SAC."""

    _attr = "q"

    def __init__(self, **kwargs):
        super().__init__()
        self._obs_dim, self.act_dim = kwargs["obs_dim"], kwargs["act_dim"]
        self._build_net([self._obs_dim + self.act_dim] + list(kwargs["hidden_sizes"]) + [1], kwargs["hidden_activation"],
                        kwargs.get("output_activation", "linear"))
        self.action_distribution_cls = kwargs["action_distribution_cls"]

    def forward(self, obs, act):
        src = obs.device
        flat = self.flat_params.sync()
        x = torch.cat([obs, act], dim=-1).detach().to(flat.device, torch.float32).contiguous()
        return torch.squeeze(self._raw(x), -1).to(src)


class ActionValueDistri(_LayerwiseNet):
    """Distributional action value: (obs, act) -> (mean, softplus(raw std)) (reference mlp.py:271-296)."""

    _attr = "q"

    def __init__(self, **kwargs):
        super().__init__()
        self._obs_dim, self.act_dim = kwargs["obs_dim"], kwargs["act_dim"]
        self._build_net([self._obs_dim + self.act_dim] + list(kwargs["hidden_sizes"]) + [2], kwargs["hidden_activation"],
                        kwargs.get("output_activation", "linear"))

    def forward(self, obs, act):
        src = obs.device
        flat = self.flat_params.sync()
        x = torch.cat([obs, act], dim=-1).detach().to(flat.device, torch.float32).contiguous()
        out = self._raw(x)
        mean, raw = torch.chunk(out, chunks=2, dim=-1)
        return torch.cat((mean, torch.nn.functional.softplus(raw)), dim=-1).to(src)


class StateValue(_FusedMlp):
    """State-value function: obs -> v (reference mlp.py:309-329)."""

    _net_attr = "v"

    def __init__(self, **kwargs):
        super().__init__()
        self._build(kwargs["obs_dim"], 1, kwargs)

    def forward(self, obs):
        return torch.squeeze(self._infer(obs, 0.0, squash=False), -1)
