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


class Stem(Conv2d):
    """The networks' stem, run by the same code as their trunk: conv 7x7/2 pad 3 (3 -> 64, + folded FixedBatchNorm) -> ReLU
    (net/resnet50.py:63-66).  x is NCHW fp32 [B,3,H,W], zero-padded on the right / bottom to Hin x Win like IRNet's crop;
    the output is NHWC [B,Ho,Wo,64].  mode 0 = SIMT fp32, 1 = 3xTF32 stem, 2 = f16x3 stem."""

    def __init__(self, weight_oihw, bn=None):
        w = np.ascontiguousarray(weight_oihw, dtype=np.float32)
        assert w.shape == (64, 3, 7, 7)
        self.cout, self.cin, self.k, self.stride, self.pad = 64, 3, 7, 2, 3
        bn4 = None if bn is None else np.ascontiguousarray(np.stack(bn), dtype=np.float32)
        self._h = ctypes.c_void_p()
        _lib.check(_lib.lib().irn_stem_create(w.ctypes.data, None if bn4 is None else bn4.ctypes.data, ctypes.byref(self._h)),
                   "irn_stem_create")

    def __call__(self, x_nchw, Hin=None, Win=None, mode=2):
        _lib.require_cuda(x_nchw)
        x = x_nchw.contiguous().float()
        B, C, H, W = x.shape
        assert C == 3
        Hin, Win = Hin or H, Win or W
        out = torch.empty((B, (Hin - 1) // 2 + 1, (Win - 1) // 2 + 1, 64), dtype=torch.float32, device=x.device)
        nbytes = _lib.lib().irn_stem_workspace_bytes(B, Hin, Win)
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            rc = _lib.lib().irn_stem_forward(self._h, _lib.ptr(x), B, H, W, Hin, Win, _lib.ptr(out), int(mode), _lib.ptr(ws), nbytes,
                                             _lib.stream_ptr())
        _lib.check(rc, "irn_stem_forward")
        return out


class ShortcutConv(Conv2d):
    """conv3 + projection shortcut of a stage's first bottleneck as the f16x3 network runs them: one K-concatenated 1x1 conv,
    relu(bn3(conv3(t2)) + bnds(ds(x sampled at `stride`))) (net/resnet50.py:46-54).  Needs planes % 64 == 0 and cin % 64 == 0.
    x NHWC [B,H,W,cin], t2 NHWC [B,Ho,Wo,planes] -> NHWC [B,Ho,Wo,4 planes]."""

    def __init__(self, w3, bn3, wds, bnds, stride):
        w3 = np.ascontiguousarray(np.asarray(w3, dtype=np.float32).reshape(len(w3), -1))
        wds = np.ascontiguousarray(np.asarray(wds, dtype=np.float32).reshape(len(wds), -1))
        self.cout, self.planes = w3.shape
        self.cin, self.stride = wds.shape[1], stride
        assert self.cout == 4 * self.planes and wds.shape[0] == self.cout
        b3, bd = (np.ascontiguousarray(np.stack(b), dtype=np.float32) for b in (bn3, bnds))
        self._h = ctypes.c_void_p()
        _lib.check(_lib.lib().irn_shortcut_conv_create(w3.ctypes.data, b3.ctypes.data, wds.ctypes.data, bd.ctypes.data, self.planes,
                                                       self.cin, stride, ctypes.byref(self._h)), "irn_shortcut_conv_create")

    def __call__(self, t2_nhwc, x_nhwc):
        _lib.require_cuda(t2_nhwc, x_nhwc)
        t2, x = t2_nhwc.contiguous().float(), x_nhwc.contiguous().float()
        B, H, W, C = x.shape
        Ho, Wo = (H - 1) // self.stride + 1, (W - 1) // self.stride + 1
        assert C == self.cin and tuple(t2.shape) == (B, Ho, Wo, self.planes)
        out = torch.empty((B, Ho, Wo, self.cout), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            rc = _lib.lib().irn_shortcut_conv_forward(self._h, _lib.ptr(t2), _lib.ptr(x), B, H, W, _lib.ptr(out), _lib.stream_ptr())
        _lib.check(rc, "irn_shortcut_conv_forward")
        return out
