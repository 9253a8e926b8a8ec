"""Flat fp32 parameter / gradient storage and the fused Adam optimizer.

The CUDA kernels take one contiguous parameter vector per network in torch `parameters()` order
(include/gops_b200.h).  `FlatParams` keeps every `nn.Parameter.data` (and `.grad`) of a module as
a VIEW into such a vector, so the modules keep the reference's `state_dict` keys and ordinary
`nn.Parameter`s while the kernels, the NCCL all-reduce and Adam work on a single buffer.
"""
import math
from typing import List, Optional

import numpy as np

import torch

from gops_b200 import _lib

GRAD_TAIL = 4  # loss, critic mean value, #done, pad -- reduced together with the gradient


class FlatParams:
    def __init__(self, module: torch.nn.Module):
        self.module = module
        self.flat = None       # [n]
        self.gbuf = None       # [n + GRAD_TAIL]; gbuf[:n] is the gradient, the tail carries scalars

    def _params(self) -> List[torch.nn.Parameter]:
        return list(self.module.parameters())

    @property
    def numel(self) -> int:
        return sum(p.numel() for p in self._params())

    def _aliased(self, buf, tensors) -> bool:
        if buf is None:
            return False
        off = 0
        base = buf.data_ptr()
        for t in tensors:
            if t is None or t.device != buf.device or t.dtype != torch.float32 or not t.is_contiguous() \
                    or t.data_ptr() != base + 4 * off:
                return False
            off += t.numel()
        return True

    def sync(self) -> torch.Tensor:
        """Make sure every parameter is a view of one flat buffer on the module's device."""
        params = self._params()
        dev = params[0].device
        if not self._aliased(self.flat, [p.data for p in params]):
            flat = torch.cat([p.data.detach().reshape(-1).to(torch.float32) for p in params]).contiguous()
            off = 0
            for p in params:
                n = p.numel()
                p.data = flat[off:off + n].view(p.shape)
                off += n
            self.flat = flat
        if self.gbuf is None or self.gbuf.device != dev or self.gbuf.numel() != self.flat.numel() + GRAD_TAIL:
            self.gbuf = torch.zeros(self.flat.numel() + GRAD_TAIL, dtype=torch.float32, device=dev)
        return self.flat

    def bind_grads(self):
        """Point every p.grad at its slice of the flat gradient buffer."""
        self.sync()
        params = self._params()
        if self._aliased(self.gbuf, [p.grad for p in params]):
            return
        off = 0
        for p in params:
            n = p.numel()
            p.grad = self.gbuf[off:off + n].view(p.shape)
            off += n

    def gather_grads(self):
        """Accept externally assigned p.grad tensors (remote_update path) into the flat buffer."""
        self.sync()
        params = self._params()
        if self._aliased(self.gbuf, [p.grad for p in params]):
            return
        off = 0
        for p in params:
            n = p.numel()
            if p.grad is None:
                self.gbuf[off:off + n].zero_()
            else:
                self.gbuf[off:off + n].copy_(p.grad.detach().reshape(-1).to(self.gbuf.device, torch.float32))
            off += n
        self.bind_grads()


class FusedAdam(torch.optim.Optimizer):
    """torch.optim.Adam semantics (no weight decay / amsgrad) executed by one CUDA kernel over the
    flat buffer (`gops_b200_adam_step`).  Being a real `Optimizer`, torch LR schedulers attach to
    it exactly as in the reference (`gops/algorithm/base.py:34-49`)."""

    def __init__(self, flat: FlatParams, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        self.flat_params = flat
        super().__init__(flat._params(), dict(lr=lr, betas=betas, eps=eps))
        self._step = 0
        self._m = None
        self._v = None

    def zero_grad(self, set_to_none: bool = False):
        if self.flat_params.gbuf is not None:
            self.flat_params.gbuf.zero_()

    def _state(self):
        fp = self.flat_params
        flat = fp.sync()
        if not flat.is_cuda:
            raise RuntimeError("gops_b200.FusedAdam: parameters must live on a CUDA device (no CPU fallback)")
        fp.gather_grads()
        self._moments(flat)
        self._step += 1
        return fp, flat

    def _moments(self, flat):
        if self._m is None or self._m.device != flat.device or self._m.numel() != flat.numel():
            self._m = torch.zeros_like(flat)
            self._v = torch.zeros_like(flat)

    @torch.no_grad()
    def multi_step_state(self):
        """(params, exp_avg, exp_avg_sq, steps taken so far, group) for a kernel that takes several Adam steps itself
        (RPI's Newton iteration, csrc/rpi.cu); `advance(n)` then records the n steps it took."""
        flat = self.flat_params.sync()
        if not flat.is_cuda:
            raise RuntimeError("gops_b200.FusedAdam: parameters must live on a CUDA device (no CPU fallback)")
        self._moments(flat)
        return flat, self._m, self._v, self._step, self.param_groups[0]

    def advance(self, n: int):
        self._step += int(n)

    @torch.no_grad()
    def fused_state(self):
        """(params, exp_avg, exp_avg_sq, step, group) of THIS step, for a kernel that applies Adam itself (the
        peer-memory gradient exchange, utils/peer_reduce.py); counts as the step."""
        _, flat = self._state()
        return flat, self._m, self._v, self._step, self.param_groups[0]

    @torch.no_grad()
    def step(self, closure=None):
        fp, flat = self._state()
        g = self.param_groups[0]
        with torch.cuda.device(flat.device):      # launch on the parameters' device and its current stream
            _lib.check(_lib.lib().gops_b200_adam_step(
                _lib.ptr(flat), _lib.ptr(fp.gbuf), _lib.ptr(self._m), _lib.ptr(self._v), flat.numel(), self._step,
                float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), _lib.stream_ptr()))


@torch.no_grad()
def polyak_update(target: FlatParams, src: FlatParams, tau: float):
    t, s = target.sync(), src.sync()
    if not t.is_cuda:
        raise RuntimeError("gops_b200.polyak_update: parameters must live on a CUDA device (no CPU fallback)")
    with torch.cuda.device(t.device):
        _lib.check(_lib.lib().gops_b200_polyak(_lib.ptr(t), _lib.ptr(s), float(tau), t.numel(), _lib.stream_ptr()))


class ScalarAdam:
    """torch.optim.Adam (default betas / eps, no weight decay) for a single fp32 scalar parameter, evaluated on the host
    with numpy float32 arithmetic in torch's operation order (torch/optim/adam.py _single_tensor_adam)."""

    def __init__(self, param: torch.nn.Parameter, lr: float, betas=(0.9, 0.999), eps: float = 1e-8):
        self.param, self.lr, self.betas, self.eps = param, lr, betas, eps
        self.step_count, self.m, self.v = 0, np.float32(0), np.float32(0)
        self.grad: Optional[float] = None

    def zero_grad(self):
        self.grad = None

    def step(self):
        if self.grad is None:
            return
        g = np.float32(self.grad)
        b1, b2 = self.betas
        self.step_count += 1
        self.m = np.float32(self.m + (g - self.m) * np.float32(1 - b1))
        self.v = np.float32(self.v * np.float32(b2) + np.float32(1 - b2) * (g * g))
        bc1, bc2 = 1 - b1 ** self.step_count, 1 - b2 ** self.step_count
        denom = np.float32(np.sqrt(self.v) / np.float32(math.sqrt(bc2)) + np.float32(self.eps))
        value = np.float32(np.float32(self.param.item()) - np.float32(self.lr / bc1) * (self.m / denom))
        with torch.no_grad():
            self.param.fill_(float(value))
