"""C1 on the device: the per-scale body of ``VOC12ClassificationDatasetMSF.__getitem__``
(voc12/dataloader.py:191-201) for decoded uint8 images that already sit in HBM.

``msf_batch(imgs_u8, scales)`` returns what the reference's loader yields per scale -- fp32 [2,3,h,w]
(image, W-flip) per image, here stacked to [2B,3,h,w] -- bit-exact with PIL's bicubic resize
(misc/imutils.py:8-22) and TorchvisionNormalize (voc12/dataloader.py:65-78), through the C ABI
(include/irn_b200.h, irn_resize_*).  JPEG decoding stays on the host.
"""
import ctypes

import numpy as np
import torch

from . import _lib

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def rescaled_size(H, W, scale):
    """misc/imutils.py:19-22 (np.round: half to even)."""
    return int(np.round(H * scale)), int(np.round(W * scale))


def resize_coeffs(in_size, out_size):
    """Pillow's 8-bit coefficient table of one axis (host): bounds int32 [out,2], kk int32 [out,ksize]."""
    L = _lib.lib()
    ks = L.irn_resize_ksize(int(in_size), int(out_size))
    if ks <= 0:
        raise _lib.IrnError("irn_resize_ksize rejected %r -> %r" % (in_size, out_size))
    bounds = np.empty((out_size, 2), np.int32)
    kk = np.empty((out_size, ks), np.int32)
    _lib.check(L.irn_resize_coeffs(int(in_size), int(out_size), bounds.ctypes.data, kk.ctypes.data), "irn_resize_coeffs")
    return bounds, kk


def normalize_lut(mean=MEAN, std=STD):
    L = _lib.lib()
    m, s = np.asarray(mean, np.float64), np.asarray(std, np.float64)
    lut = np.empty((3, 256), np.float32)
    _lib.check(L.irn_normalize_lut(m.ctypes.data, s.ctypes.data, lut.ctypes.data), "irn_normalize_lut")
    return lut


class _Plan:
    def __init__(self, H, W, oh, ow, mean, std):
        L = _lib.lib()
        m, s = np.asarray(mean, np.float64), np.asarray(std, np.float64)
        h = ctypes.c_void_p()
        _lib.check(L.irn_resize_plan_create(H, W, oh, ow, m.ctypes.data, s.ctypes.data, ctypes.byref(h)), "irn_resize_plan_create")
        self.handle, self.shape = h, (H, W, oh, ow)

    def __del__(self):
        try:
            if self.handle:
                _lib.lib().irn_resize_plan_destroy(self.handle)
        except Exception:
            pass


_plans = {}
_ws = {}


def _plan(dev, H, W, oh, ow, mean, std):
    key = (dev.index, H, W, oh, ow, tuple(mean), tuple(std))
    if key not in _plans and len(_plans) >= 1024:      # VOC has a few hundred distinct sizes x scales; bound the cache anyway
        _plans.clear()
    if key not in _plans:
        with torch.cuda.device(dev):
            _plans[key] = _Plan(H, W, oh, ow, mean, std)
    return _plans[key]


def resize_normalize(imgs_u8, out_hw, mean=MEAN, std=STD, want_u8=False, out=None):
    """imgs_u8: cuda uint8 [B,H,W,3] (or [H,W,3]).  Returns fp32 [2B,3,oh,ow] (rows 2b, 2b+1 = image b, its W-flip)
    and, with want_u8, also the resized uint8 [B,oh,ow,3]."""
    _lib.require_cuda(imgs_u8)
    if imgs_u8.dtype != torch.uint8 or imgs_u8.shape[-1] != 3:
        raise _lib.IrnError("resize_normalize: expected uint8 [...,H,W,3], got %s %s" % (imgs_u8.dtype, tuple(imgs_u8.shape)))
    x = imgs_u8.reshape((-1,) + tuple(imgs_u8.shape[-3:])).contiguous()
    B, H, W, _ = x.shape
    oh, ow = int(out_hw[0]), int(out_hw[1])
    dev = x.device
    L = _lib.lib()
    plan = _plan(dev, H, W, oh, ow, mean, std)
    if out is None:
        out = torch.empty((2 * B, 3, oh, ow), dtype=torch.float32, device=dev)
    elif tuple(out.shape) != (2 * B, 3, oh, ow) or out.dtype != torch.float32 or not out.is_contiguous():
        raise _lib.IrnError("resize_normalize: bad output buffer")
    u8 = torch.empty((B, oh, ow, 3), dtype=torch.uint8, device=dev) if want_u8 else None
    need = L.irn_resize_workspace_bytes(plan.handle, B)
    ws = _ws.get(dev.index)
    if ws is None or ws.numel() < need:
        ws = torch.empty(int(need * 1.25) + 256, dtype=torch.uint8, device=dev)
        _ws[dev.index] = ws
    with torch.cuda.device(dev):
        rc = L.irn_resize_forward(plan.handle, _lib.ptr(x), B, _lib.ptr(out), _lib.ptr(u8), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
    _lib.check(rc, "irn_resize_forward")
    return (out, u8) if want_u8 else out


def msf_batch(imgs_u8, scales, mean=MEAN, std=STD):
    """voc12/dataloader.py:191-201 for a batch of equal-sized images: list (one entry per scale) of fp32 [2B,3,h_s,w_s]."""
    H, W = int(imgs_u8.shape[-3]), int(imgs_u8.shape[-2])
    return [resize_normalize(imgs_u8, (H, W) if s == 1 else rescaled_size(H, W, s), mean, std) for s in scales]


def resize_normalize_ragged(flat_u8, sizes, scale):
    """One scale of the pyramids of images of different sizes in one call: flat_u8 cuda uint8 holding the images uint8 [H_i,W_i,3]
    back to back (StepContext.pack_images), sizes [(H_i, W_i)].  Returns (canvas fp32 [2P,3,Hc,Wc], [(h_i, w_i)]): image i resized to
    (h_i, w_i) = rescaled_size(H_i, W_i, scale) (itself at scale 1.0) at the top-left corner of rows 2i (as is) and 2i+1 (W-flipped
    within w_i), +0.0 elsewhere; (Hc, Wc) the largest (h_i, w_i).  Each corner equals resize_normalize of that image alone, bit for bit
    (the loader's MEAN / STD normalisation)."""
    from .indexing import _workspace
    from .irn import _normalize_lut
    _lib.require_cuda(flat_u8)
    sizes = [(int(h), int(w)) for h, w in sizes]
    P = len(sizes)
    if P == 0:
        raise _lib.IrnError("resize_normalize_ragged: empty batch")
    if flat_u8.dtype != torch.uint8 or flat_u8.dim() != 1 or not flat_u8.is_contiguous():
        raise _lib.IrnError("resize_normalize_ragged: expected one flat contiguous uint8 buffer, got %s %s" % (flat_u8.dtype, tuple(flat_u8.shape)))
    out_hw = [(H, W) if scale == 1 else rescaled_size(H, W, scale) for H, W in sizes]
    hw = np.ascontiguousarray(np.asarray(sizes, np.int32).reshape(P, 2))
    ohw = np.ascontiguousarray(np.asarray(out_hw, np.int32).reshape(P, 2))
    offs = np.zeros(P, np.int64)
    np.cumsum(hw[:-1, 0].astype(np.int64) * hw[:-1, 1] * 3, out=offs[1:])
    Hc, Wc = int(ohw[:, 0].max()), int(ohw[:, 1].max())
    dev = flat_u8.device
    L = _lib.lib()
    out = torch.empty((2 * P, 3, Hc, Wc), dtype=torch.float32, device=dev)
    ws = _workspace(L.irn_resize_ragged_workspace_bytes(hw.ctypes.data, ohw.ctypes.data, P), dev)
    with torch.cuda.device(dev):
        rc = L.irn_resize_ragged_forward(_lib.ptr(flat_u8), flat_u8.numel(), offs.ctypes.data, hw.ctypes.data, ohw.ctypes.data, P, Hc, Wc,
                                         _lib.ptr(_normalize_lut(dev)), _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
    _lib.check(rc, "irn_resize_ragged_forward")
    return out, out_hw
