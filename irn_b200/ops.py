"""Single-operator access to libirn_b200 (unit tests, wiring other topologies)."""
import ctypes

import numpy as np
import torch

from . import _lib


class Conv2d:
    """conv (+ folded FixedBatchNorm) -> [+ residual] -> [ReLU] on NHWC fp32 CUDA tensors
    (net/resnet50.py:34-54 building block).  mode 0 = SIMT fp32, 1 = wgmma 3xTF32, 2 = wgmma f16x3."""

    def __init__(self, weight_oihw, bn=None, stride=1, pad=0):
        w = np.ascontiguousarray(weight_oihw, dtype=np.float32)
        self.cout, self.cin, self.k, _ = w.shape
        self.stride, self.pad = stride, pad
        bn4 = None if bn is None else np.ascontiguousarray(np.stack(bn), dtype=np.float32)
        self._h = ctypes.c_void_p()
        _lib.check(_lib.lib().irn_conv_create(w.ctypes.data, None if bn4 is None else bn4.ctypes.data, self.cin, self.cout, self.k,
                                              stride, pad, ctypes.byref(self._h)), "irn_conv_create")

    def __del__(self):
        try:
            if self._h:
                _lib.lib().irn_conv_destroy(self._h)
        except Exception:
            pass

    def __call__(self, x_nhwc, residual=None, relu=False, mode=1):
        _lib.require_cuda(x_nhwc, residual)
        x = x_nhwc.contiguous().float()
        B, H, W, C = x.shape
        assert C == self.cin
        Ho = (H + 2 * self.pad - self.k) // self.stride + 1
        Wo = (W + 2 * self.pad - self.k) // self.stride + 1
        out = torch.empty((B, Ho, Wo, self.cout), dtype=torch.float32, device=x.device)
        res = None if residual is None else residual.contiguous().float()
        with torch.cuda.device(x.device):
            rc = _lib.lib().irn_conv_forward(self._h, _lib.ptr(x), B, H, W, _lib.ptr(res), _lib.ptr(out), int(relu), int(mode), _lib.stream_ptr())
        _lib.check(rc, "irn_conv_forward")
        return out
