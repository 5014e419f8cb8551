"""Drop-in for ``net.resnet50_cam`` -- select with ``--cam_network irn_b200.cam``.

``CAM`` keeps the reference's construction / ``load_state_dict(strict=True)`` / ``eval()`` /
``cuda()`` / ``__call__`` protocol (step/make_cam.py:63-65,24,35) and its checkpoint keys
(SURVEY.md D10), but the forward pass is libirn_b200's native plan (irn_cam_forward):
BN-folded NHWC convolutions, fused ReLU/residual epilogues and the fused CAM head
(relu(conv1x1) of the image + flipped image, net/resnet50_cam.py:65-68).
"""
import ctypes

import torch

from . import _lib, _pack
from ._params import CamParams
from .indexing import _workspace


class _Plan:
    """Owns an irn_net handle on one device."""

    def __init__(self, handle, device):
        self.handle, self.device = handle, device

    def __del__(self):
        try:
            if self.handle:
                _lib.lib().irn_net_destroy(self.handle)
        except Exception:
            pass


class CAM(CamParams):
    def __init__(self):
        super().__init__()
        self._plan = None
        self._conv_mode = None      # None = the library's default for this network

    def set_conv_mode(self, mode):
        """Convolution arithmetic of the native plan: 0 SIMT fp32, 1 wgmma 3xTF32, 2 wgmma f16x3 (irn_net_set_conv_mode)."""
        self._conv_mode = None if mode is None else int(mode)
        if self._plan is not None and self._conv_mode is not None:
            _lib.check(_lib.lib().irn_net_set_conv_mode(self._plan.handle, self._conv_mode), "irn_net_set_conv_mode")
        return self

    # the reference's Net.train() ignores `mode` (net/resnet50_cam.py:39-43); inference only here
    def train(self, mode=True):
        return self

    def _invalidate(self):
        self._plan = None

    def load_state_dict(self, *a, **k):
        self._invalidate()
        return super().load_state_dict(*a, **k)

    def _get_plan(self, device):
        if self._plan is None or self._plan.device != device:
            blob = _pack.pack_cam(self.state_dict())
            h = ctypes.c_void_p()
            with torch.cuda.device(device):
                _lib.check(_lib.lib().irn_cam_net_create(blob.ctypes.data, blob.size, ctypes.byref(h)), "irn_cam_net_create")
            self._plan = _Plan(h, device)
            if self._conv_mode is not None:
                _lib.check(_lib.lib().irn_net_set_conv_mode(h, self._conv_mode), "irn_net_set_conv_mode")
        return self._plan

    def forward_batch(self, x):
        """x cuda fp32 [2P,3,H,W] (P image/flip pairs of equal size) -> [P,20,ceil(H/16),ceil(W/16)]."""
        _lib.require_cuda(x)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[0] % 2:
            raise _lib.IrnError("CAM expects [2P,3,H,W] (image, flipped image) pairs, got %s" % (tuple(x.shape),))
        x = x.contiguous().float()
        B, _, H, W = x.shape
        L = _lib.lib()
        plan = self._get_plan(x.device)
        h, w = (H - 1) // 16 + 1, (W - 1) // 16 + 1
        out = torch.empty((B // 2, 20, h, w), dtype=torch.float32, device=x.device)
        need = L.irn_cam_workspace_bytes(B, H, W)
        ws = _workspace(need, x.device)
        with torch.cuda.device(x.device):
            rc = L.irn_cam_forward(plan.handle, _lib.ptr(x), B, H, W, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "irn_cam_forward")
        return out

    def forward(self, x):
        """Reference signature (net/resnet50_cam.py:55-70): [2,3,h,w] -> [20,ceil(h/16),ceil(w/16)]."""
        return self.forward_batch(x)[0]


Net = CAM   # `net.resnet50_cam.Net` is the train-time classifier (out of scope); kept as an alias for importers
