"""C4 host wrapper: multi-scale CAM merge through the C ABI (step/make_cam.py:38-52)."""
import ctypes

import numpy as np
import torch

from . import _lib
from ._params import MAX_CLASSES


_scratches = {}


def _scratch(dev):
    """2 x K <= 2 x 128 per-class maxima (int-ordered float bits); one persistent buffer per device, reused in stream order."""
    key = dev.index
    if key not in _scratches:
        _scratches[key] = torch.empty(2 * MAX_CLASSES, dtype=torch.int32, device=dev)
    return _scratches[key]


def merge_cams(outputs, size, label, want_highres=True):
    """outputs: list of cuda fp32 [C,h_s,w_s] (one per scale); size=(H,W); label: fp32[C] multi-hot (any device).
    Returns (keys LongTensor[K] on cpu, strided_cam cuda [K,ceil(H/4),ceil(W/4)], highres_cam cuda [K,H,W] or None)."""
    L = _lib.lib()
    _lib.require_cuda(*outputs)
    dev = outputs[0].device
    outs = [o.contiguous().float() for o in outputs]
    H, W = int(size[0]), int(size[1])
    keys = torch.nonzero(torch.as_tensor(label).cpu())[:, 0]          # step/make_cam.py:46
    K = int(keys.numel())
    h4, w4 = (H - 1) // 4 + 1, (W - 1) // 4 + 1
    strided = torch.empty((K, h4, w4), dtype=torch.float32, device=dev)
    highres = torch.empty((K, H, W), dtype=torch.float32, device=dev) if want_highres else None
    if K == 0:
        return keys, strided, highres
    n = len(outs)
    ptrs = (ctypes.c_void_p * n)(*[o.data_ptr() for o in outs])
    hs = (ctypes.c_int * n)(*[int(o.shape[1]) for o in outs])
    ws = (ctypes.c_int * n)(*[int(o.shape[2]) for o in outs])
    keys_host = np.ascontiguousarray(keys.numpy().astype(np.int32))
    scratch = _scratch(dev)
    with torch.cuda.device(dev):
        rc = L.irn_cam_merge_classes(ptrs, hs, ws, n, int(outs[0].shape[0]), H, W, keys_host.ctypes.data, K, _lib.ptr(strided),
                                     _lib.ptr(highres), _lib.ptr(scratch), _lib.stream_ptr())
    _lib.check(rc, "irn_cam_merge")
    return keys, strided, highres
