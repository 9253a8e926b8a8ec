"""Host-side handle of the layer-wise wgmma MLP (C ABI `gops_b200_mlpnet_*`, csrc/dense_tc.cu): forward / backward of an
`mlp()` network (reference gops/apprfunc/mlp.py:36-41) of any depth with widths <= 256, evaluated on the tensor cores in
BF16x3 (FP32-accurate) arithmetic.  Plumbing only: device buffers are torch tensors, the arithmetic is in the library."""
import ctypes as C
from typing import Optional, Sequence

import torch

from gops_b200 import _lib


class LayerwiseMlp:
    def __init__(self, sizes: Sequence[int], hidden_activation: str, max_batch: int, slots: int = 1, device=None):
        self.sizes = [int(s) for s in sizes]
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.max_batch, self.slots = int(max_batch), int(slots)
        arr = (C.c_int32 * len(self.sizes))(*self.sizes)
        self.handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().gops_b200_mlpnet_create(arr, len(self.sizes), _lib.ACT_IDS[hidden_activation],
                                                         self.max_batch, self.slots, C.byref(self.handle)))
        self.nparam = int(_lib.lib().gops_b200_mlpnet_param_count(self.handle))
        self._params = None

    def __del__(self):
        try:
            if self.handle:
                _lib.lib().gops_b200_mlpnet_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def pack(self, params_flat: torch.Tensor):
        """Split the current weights into bf16 planes (once per parameter update)."""
        assert params_flat.is_cuda and params_flat.dtype == torch.float32 and params_flat.numel() == self.nparam
        self._params = params_flat            # biases are read from this vector by the forward kernels
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().gops_b200_mlpnet_pack(self.handle, _lib.ptr(params_flat), _lib.stream_ptr()))

    def forward(self, x: torch.Tensor, slot: int = 0, train: bool = True, out: Optional[torch.Tensor] = None):
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
        B = x.shape[0]
        y = out if out is not None else torch.empty((B, self.sizes[-1]), dtype=torch.float32, device=x.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().gops_b200_mlpnet_forward(self.handle, _lib.ptr(x), x.stride(0), B, slot, int(train),
                                                          _lib.ptr(y), y.stride(0), _lib.stream_ptr()))
        return y

    def backward(self, dy: torch.Tensor, slot: int = 0, grad: Optional[torch.Tensor] = None, accumulate: bool = False,
                 want_dx: bool = False):
        assert dy.is_cuda and dy.dtype == torch.float32 and dy.dim() == 2 and dy.stride(1) == 1
        B = dy.shape[0]
        dx = torch.empty((B, self.sizes[0]), dtype=torch.float32, device=dy.device) if want_dx else None
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().gops_b200_mlpnet_backward(
                self.handle, _lib.ptr(dy), dy.stride(0), B, slot, _lib.ptr(grad), int(accumulate), _lib.ptr(dx),
                dx.stride(0) if dx is not None else 0, _lib.stream_ptr()))
        return dx


class LayerwiseMlpPair:
    """Two `LayerwiseMlp` handles of identical shape (twin critics) evaluated on one shared input with paired passes
    (`gops_b200_mlpnet_pair_*`): every layer launch runs both networks, each with the arithmetic of its single pass."""

    def __init__(self, a: LayerwiseMlp, b: LayerwiseMlp):
        self.a, self.b = a, b
        self.device = a.device

    def forward(self, x: torch.Tensor, slot: int = 0, train: bool = True, out_a: Optional[torch.Tensor] = None,
                out_b: Optional[torch.Tensor] = None):
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
        B, n = x.shape[0], self.a.sizes[-1]
        ya = out_a if out_a is not None else torch.empty((B, n), dtype=torch.float32, device=x.device)
        yb = out_b if out_b is not None else torch.empty((B, n), dtype=torch.float32, device=x.device)
        assert ya.stride(0) == yb.stride(0) and ya.stride(1) == 1 and yb.stride(1) == 1
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().gops_b200_mlpnet_pair_forward(
                self.a.handle, self.b.handle, _lib.ptr(x), x.stride(0), B, slot, int(train), _lib.ptr(ya), _lib.ptr(yb),
                ya.stride(0), _lib.stream_ptr()))
        return ya, yb

    def backward(self, dy_a: torch.Tensor, dy_b: torch.Tensor, slot: int = 0, grad_a: Optional[torch.Tensor] = None,
                 grad_b: Optional[torch.Tensor] = None, accumulate: bool = False, want_dx: bool = False):
        for dy in (dy_a, dy_b):
            assert dy.is_cuda and dy.dtype == torch.float32 and dy.dim() == 2 and dy.stride(1) == 1
        assert dy_a.shape == dy_b.shape and dy_a.stride(0) == dy_b.stride(0)
        B = dy_a.shape[0]
        dx_a = dx_b = None
        if want_dx:
            dx_a = torch.empty((B, self.a.sizes[0]), dtype=torch.float32, device=dy_a.device)
            dx_b = torch.empty_like(dx_a)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().gops_b200_mlpnet_pair_backward(
                self.a.handle, self.b.handle, _lib.ptr(dy_a), _lib.ptr(dy_b), dy_a.stride(0), B, slot, _lib.ptr(grad_a),
                _lib.ptr(grad_b), int(accumulate), _lib.ptr(dx_a), _lib.ptr(dx_b),
                dx_a.stride(0) if dx_a is not None else 0, _lib.stream_ptr()))
        return dx_a, dx_b


def layerwise_pair(a, b, max_batch: int, slots: int, tag: str) -> LayerwiseMlpPair:
    """The library handles of two `_LayerwiseNet` modules of identical shape (twin critics), sized alike so that they
    can run as a pair."""
    na, nb = a.layerwise(max_batch, slots, tag), b.layerwise(max_batch, slots, tag)
    if (na.max_batch, na.slots) != (nb.max_batch, nb.slots):
        mb, sl = max(na.max_batch, nb.max_batch), max(na.slots, nb.slots)
        na, nb = a.layerwise(mb, sl, tag), b.layerwise(mb, sl, tag)
    return LayerwiseMlpPair(na, nb)
