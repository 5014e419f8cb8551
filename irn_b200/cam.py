"""Drop-in for ``net.resnet50_cam`` -- select with ``--cam_network irn_b200.cam``.

``CAM`` keeps the reference's construction / ``load_state_dict(strict=True)`` / ``eval()`` /
``cuda()`` / ``__call__`` protocol (step/make_cam.py:63-65,24,35) and its checkpoint keys
(SURVEY.md D10), but the forward pass is libirn_b200's native plan (irn_cam_forward):
BN-folded NHWC convolutions, fused ReLU/residual epilogues and the fused CAM head
(relu(conv1x1) of the image + flipped image, net/resnet50_cam.py:65-68).
"""
import ctypes

import numpy as np
import torch

from . import _lib, _pack
from ._params import MAX_CLASSES, CamParams
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

    def set_tap(self, tap_id, dst):
        """irn_net_set_tap: the plan's forwards copy tap `tap_id` into `dst` (contiguous fp32 on the plan's device); None clears it."""
        if dst is not None:
            _lib.require_cuda(dst)
            if dst.dtype != torch.float32 or not dst.is_contiguous() or dst.device != self.device:
                raise _lib.IrnError("a tap buffer is a contiguous fp32 tensor on %s" % self.device)
        _lib.check(_lib.lib().irn_net_set_tap(self.handle, int(tap_id), _lib.ptr(dst), 0 if dst is None else dst.numel() * 4),
                   "irn_net_set_tap")


def tap_shape(kind, tap_id, B, H=0, W=0, crop_size=0, n_classes=20):
    """NHWC shape of tap `tap_id` (irn_net_tap_shape) for a forward of B samples: kind 0 = CAM of `n_classes` classes on H x W,
    1 = IRNet on crop_size."""
    shape = (ctypes.c_int * 4)()
    if kind == 0 and n_classes != 20:
        _lib.check(_lib.lib().irn_cam_tap_shape(int(n_classes), int(tap_id), int(B), int(H), int(W), shape), "irn_cam_tap_shape")
    else:
        _lib.check(_lib.lib().irn_net_tap_shape(int(kind), int(tap_id), int(B), int(H), int(W), int(crop_size), shape),
                   "irn_net_tap_shape")
    return tuple(shape)


class CAM(CamParams):
    """The class count C follows the checkpoint: load_state_dict takes it from `classifier.weight` ([C,2048,1,1], 1 <= C <= 128;
    20 for PASCAL VOC, 80 for MS COCO), and every forward returns C CAM planes per image."""

    def __init__(self, n_classes=20):
        super().__init__(n_classes)
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

    def set_tap(self, tap_id, dst, device=None):
        """Test instrumentation: from now on, forwards copy layer tap `tap_id` (the IRN_TAP_* ids of include/irn_b200.h) into `dst`,
        a contiguous fp32 cuda tensor of tap_shape(0, tap_id, ...) elements or more; dst None clears the tap.  Taps belong to the
        current plan: load_state_dict drops them."""
        dev = dst.device if dst is not None else (device or torch.device("cuda", torch.cuda.current_device()))
        self._get_plan(dev).set_tap(tap_id, dst)
        return self

    def _invalidate(self):
        self._plan = None

    @property
    def n_classes(self):
        return int(self.classifier.weight.shape[0])

    def load_state_dict(self, state_dict, *a, **k):
        self._invalidate()
        w = state_dict.get("classifier.weight") if hasattr(state_dict, "get") else None
        if w is not None and tuple(w.shape[1:]) == (2048, 1, 1) and int(w.shape[0]) != self.n_classes:
            C = int(w.shape[0])
            if not 1 <= C <= MAX_CLASSES:
                raise _lib.IrnError("CAM checkpoint has a %d-class classifier; 1..%d classes are supported" % (C, MAX_CLASSES))
            self.classifier = torch.nn.Conv2d(2048, C, 1, bias=False)
            self.newly_added = torch.nn.ModuleList([self.classifier])
        return super().load_state_dict(state_dict, *a, **k)

    def _get_plan(self, device):
        if self._plan is None or self._plan.device != device:
            blob = _pack.pack_cam(self.state_dict())
            h = ctypes.c_void_p()
            with torch.cuda.device(device):
                _lib.check(_lib.lib().irn_cam_net_create_classes(blob.ctypes.data, blob.size, self.n_classes, ctypes.byref(h)),
                           "irn_cam_net_create")
            self._plan = _Plan(h, device)
            if self._conv_mode is not None:
                _lib.check(_lib.lib().irn_net_set_conv_mode(h, self._conv_mode), "irn_net_set_conv_mode")
        return self._plan

    def forward_batch(self, x):
        """x cuda fp32 [2P,3,H,W] (P image/flip pairs of equal size) -> [P,C,ceil(H/16),ceil(W/16)]."""
        _lib.require_cuda(x)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[0] % 2:
            raise _lib.IrnError("CAM expects [2P,3,H,W] (image, flipped image) pairs, got %s" % (tuple(x.shape),))
        x = x.contiguous().float()
        B, _, H, W = x.shape
        L = _lib.lib()
        plan = self._get_plan(x.device)
        h, w = (H - 1) // 16 + 1, (W - 1) // 16 + 1
        out = torch.empty((B // 2, self.n_classes, h, w), dtype=torch.float32, device=x.device)
        need = L.irn_cam_workspace_bytes_classes(B, H, W, self.n_classes)
        ws = _workspace(need, x.device)
        with torch.cuda.device(x.device):
            rc = L.irn_cam_forward(plan.handle, _lib.ptr(x), B, H, W, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "irn_cam_forward")
        return out

    def forward_ragged(self, canvas, extents):
        """Pairs of different sizes in one forward: canvas cuda fp32 [2P,3,Hc,Wc] with pair i's image and its flip of extents[i] =
        (h_i, w_i) pixels at the top-left corner and +0.0 elsewhere (preprocess.resize_normalize_ragged) -> [P,C,ceil(Hc/16),ceil(Wc/16)]:
        pair i's ceil(h_i/16) x ceil(w_i/16) corner equals, bit for bit, forward_batch of that pair alone; the rest is 0."""
        _lib.require_cuda(canvas)
        if canvas.dim() != 4 or canvas.shape[1] != 3 or canvas.shape[0] % 2 or canvas.dtype != torch.float32:
            raise _lib.IrnError("CAM.forward_ragged expects fp32 [2P,3,Hc,Wc] (image, flipped image) pairs, got %s %s" %
                                (canvas.dtype, tuple(canvas.shape)))
        x = canvas.contiguous()
        B, _, H, W = x.shape
        hw = np.ascontiguousarray(np.asarray(extents, dtype=np.int32).reshape(-1, 2))
        if hw.shape[0] != B // 2:
            raise _lib.IrnError("CAM.forward_ragged: %d extents for %d pairs" % (hw.shape[0], B // 2))
        L = _lib.lib()
        plan = self._get_plan(x.device)
        out = torch.empty((B // 2, self.n_classes, (H - 1) // 16 + 1, (W - 1) // 16 + 1), dtype=torch.float32, device=x.device)
        ws = _workspace(L.irn_cam_workspace_bytes_classes(B, H, W, self.n_classes), x.device)
        with torch.cuda.device(x.device):
            rc = L.irn_cam_forward_ragged(plan.handle, _lib.ptr(x), B, H, W, hw.ctypes.data, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                          _lib.stream_ptr())
        _lib.check(rc, "irn_cam_forward_ragged")
        return out

    def forward(self, x):
        """Reference signature (net/resnet50_cam.py:55-70): [2,3,h,w] -> [C,ceil(h/16),ceil(w/16)]."""
        return self.forward_batch(x)[0]


Net = CAM   # `net.resnet50_cam.Net` is the train-time classifier (out of scope); kept as an alias for importers
