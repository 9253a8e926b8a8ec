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
