"""Drop-in for ``net.resnet50_irn`` -- select with ``--irn_network irn_b200.irn``.

``EdgeDisplacement`` keeps the reference protocol (construction, ``load_state_dict(strict=False)``,
``eval()``, ``cuda()``, ``__call__([2,3,H,W]) -> (edge [1,h,w], dp [2,h,w])``;
step/make_sem_seg_labels.py:58-60,32) and checkpoint keys; the forward pass is libirn_b200's
native plan (irn_edge_displacement_forward).  MeanShift is always applied (the label steps run the
model in eval mode, net/resnet50_irn.py:105-108).
"""
import ctypes

import torch

from . import _lib, _pack
from ._params import IrnParams
from .cam import _Plan
from .indexing import _workspace


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

    def forward(self, x):
        """Reference signature (net/resnet50_irn.py:223-234): [2,3,H,W] -> (edge [1,h,w], dp [2,h,w])."""
        if x.dim() != 4 or tuple(x.shape[:2]) != (2, 3):
            raise _lib.IrnError("EdgeDisplacement expects [2,3,H,W] (image, flipped image), got %s" % (tuple(x.shape),))
        e, d = self.forward_batch(x)
        return e[0], d[0]
