"""Drop-in for ``net.resnet50_irn`` -- select with ``--irn_network irn_b200.irn``.

``EdgeDisplacement`` keeps the reference protocol (construction, ``load_state_dict(strict=False)``,
``eval()``, ``cuda()``, ``__call__([2,3,H,W]) -> (edge [1,h,w], dp [2,h,w])``;
step/make_sem_seg_labels.py:58-60,32) and checkpoint keys; the forward pass is libirn_b200's
native plan (irn_edge_displacement_forward).  MeanShift is always applied (the label steps run the
model in eval mode, net/resnet50_irn.py:105-108).
"""
import ctypes

import numpy as np
import torch

from . import _lib, _pack, preprocess
from ._params import IrnParams
from .cam import _Plan
from .indexing import _workspace

_luts = {}


def _normalize_lut(device):
    """The loader's normalisation table (irn_normalize_lut) on `device`, uploaded once."""
    t = _luts.get(device)
    if t is None:
        t = torch.from_numpy(preprocess.normalize_lut()).to(device)
        _luts[device] = t
    return t


class EdgeDisplacement(IrnParams):
    def __init__(self, crop_size=512, stride=4):
        super().__init__()
        self.crop_size = crop_size
        self.stride = stride
        self._plan = None
        self._conv_mode = None

    def set_conv_mode(self, mode):
        """0 SIMT fp32, 1 wgmma 3xTF32, 2 wgmma f16x3 (default)."""
        self._conv_mode = None if mode is None else int(mode)
        if self._plan is not None and self._conv_mode is not None:
            _lib.check(_lib.lib().irn_net_set_conv_mode(self._plan.handle, self._conv_mode), "irn_net_set_conv_mode")
        return self

    def set_tap(self, tap_id, dst, device=None):
        """Test instrumentation, as CAM.set_tap: forwards copy tap `tap_id` (shape: cam.tap_shape(1, tap_id, 2P, crop_size=...))
        into `dst`; None clears it."""
        dev = dst.device if dst is not None else (device or torch.device("cuda", torch.cuda.current_device()))
        self._get_plan(dev).set_tap(tap_id, dst)
        return self

    def load_state_dict(self, *a, **k):
        self._plan = None
        return super().load_state_dict(*a, **k)

    def _get_plan(self, device):
        if self._plan is None or self._plan.device != device:
            blob = _pack.pack_irn(self.state_dict())
            h = ctypes.c_void_p()
            with torch.cuda.device(device):
                _lib.check(_lib.lib().irn_irn_net_create(blob.ctypes.data, blob.size, ctypes.byref(h)), "irn_irn_net_create")
            self._plan = _Plan(h, device)
            if self._conv_mode is not None:
                _lib.check(_lib.lib().irn_net_set_conv_mode(h, self._conv_mode), "irn_net_set_conv_mode")
        return self._plan

    def forward_batch(self, x):
        """x cuda fp32 [2P,3,H,W] -> (edge [P,1,fh,fw], dp [P,2,fh,fw])."""
        _lib.require_cuda(x)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[0] % 2:
            raise _lib.IrnError("EdgeDisplacement expects [2P,3,H,W] (image, flipped image) pairs, got %s" % (tuple(x.shape),))
        if self.stride != 4:
            raise _lib.IrnError("EdgeDisplacement: only stride=4 (the reference default) is built")
        x = x.contiguous().float()
        P, H, W = int(x.shape[0]) // 2, int(x.shape[2]), int(x.shape[3])
        L = _lib.lib()
        plan = self._get_plan(x.device)
        fh, fw = (H - 1) // 4 + 1, (W - 1) // 4 + 1
        edge = torch.empty((P, 1, fh, fw), dtype=torch.float32, device=x.device)
        dp = torch.empty((P, 2, fh, fw), dtype=torch.float32, device=x.device)
        need = L.irn_edge_displacement_workspace_bytes(P, H, W, int(self.crop_size))
        if need == 0:
            raise _lib.IrnError("EdgeDisplacement: image %dx%d exceeds crop_size %d" % (H, W, self.crop_size))
        ws = _workspace(need, x.device)
        with torch.cuda.device(x.device):
            rc = L.irn_edge_displacement_forward(plan.handle, _lib.ptr(x), P, H, W, int(self.crop_size), _lib.ptr(edge), _lib.ptr(dp),
                                                 _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "irn_edge_displacement_forward")
        return edge, dp

    def forward_ragged(self, images, sizes=None):
        """P decoded images of any sizes <= crop_size in one forward: `images` is a list of uint8 [H_i,W_i,3] RGB tensors, or one
        flat uint8 cuda tensor holding them back to back with `sizes` = [(H_i, W_i)].  Returns (edge [P,1,fc,fc], dp [P,2,fc,fc]),
        fc = (crop_size-1)//4+1: image i's ceil(H_i/4) x ceil(W_i/4) corner equals, bit for bit, forward_batch of its scale-1.0
        (image, flipped image) pair alone; elsewhere edge is 1.0 and dp 0 (the random walk's padding)."""
        if self.stride != 4:
            raise _lib.IrnError("EdgeDisplacement: only stride=4 (the reference default) is built")
        if sizes is None:
            sizes = [(int(t.shape[0]), int(t.shape[1])) for t in images]
            flat = torch.cat([t.reshape(-1) for t in images]) if len(images) > 1 else images[0].reshape(-1)
        else:
            flat = images
        sizes = [(int(h), int(w)) for h, w in sizes]
        P = len(sizes)
        if P == 0:
            raise _lib.IrnError("EdgeDisplacement.forward_ragged: empty batch")
        S = int(self.crop_size)
        for i, (h, w) in enumerate(sizes):
            if max(h, w) > S:
                raise _lib.IrnError("EdgeDisplacement: image %d is %dx%d, larger than crop_size %d (--irn_crop_size)" % (i, h, w, S))
        if flat.dtype != torch.uint8 or flat.dim() != 1:
            raise _lib.IrnError("EdgeDisplacement.forward_ragged expects uint8 images, got %s %s" % (flat.dtype, tuple(flat.shape)))
        dev = torch.device("cuda", torch.cuda.current_device()) if not flat.is_cuda else flat.device
        flat = flat.to(dev, non_blocking=True).contiguous()
        hw = np.ascontiguousarray(np.asarray(sizes, dtype=np.int32).reshape(P, 2))
        offs = np.zeros(P, np.int64)
        np.cumsum(hw[:-1, 0].astype(np.int64) * hw[:-1, 1] * 3, out=offs[1:])
        L = _lib.lib()
        plan = self._get_plan(dev)
        fc = (S - 1) // 4 + 1
        edge = torch.empty((P, 1, fc, fc), dtype=torch.float32, device=dev)
        dp = torch.empty((P, 2, fc, fc), dtype=torch.float32, device=dev)
        ws = _workspace(L.irn_edge_displacement_ragged_workspace_bytes(P, S), dev)
        with torch.cuda.device(dev):
            rc = L.irn_edge_displacement_forward_ragged(plan.handle, _lib.ptr(flat), flat.numel(), offs.ctypes.data, hw.ctypes.data, P, S,
                                                        _lib.ptr(_normalize_lut(dev)), _lib.ptr(edge), _lib.ptr(dp), _lib.ptr(ws),
                                                        ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "irn_edge_displacement_forward_ragged")
        return edge, dp

    def forward(self, x):
        """Reference signature (net/resnet50_irn.py:223-234): [2,3,H,W] -> (edge [1,h,w], dp [2,h,w])."""
        if x.dim() != 4 or tuple(x.shape[:2]) != (2, 3):
            raise _lib.IrnError("EdgeDisplacement expects [2,3,H,W] (image, flipped image), got %s" % (tuple(x.shape),))
        e, d = self.forward_batch(x)
        return e[0], d[0]
