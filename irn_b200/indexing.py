"""Drop-in for the reference's ``misc/indexing.py`` on H100.

Same names, argument meaning and return layout as the reference (misc/indexing.py:6-167):
``PathIndex`` (identical public attributes, built by the C ABI on the host, integer
bit-exact) and ``propagate_to_edge(x, edge, radius=5, beta=10, exp_times=8)``.  The dense
(hw)^2 transition matrix of the reference is never formed: libirn_b200's stencil kernels
iterate the same operator 2**exp_times times (include/irn_b200.h, irn_random_walk).
"""
import ctypes

import numpy as np
import torch

from . import _lib


class PathIndex:
    """misc/indexing.py:6-88.  Attributes: radius, radius_floor, search_paths (list of int64
    [n_paths, L, 2]), search_dst (int64 [n_dst, 2]), path_indices (list of int64
    [n_paths, L, n_src]), src_indices (int64 [n_src]), dst_indices (int64 [n_dst, n_src])."""

    def __init__(self, radius, default_size):
        L = _lib.lib()
        if int(radius) != radius:
            raise _lib.IrnError("PathIndex: integer radius required, got %r" % (radius,))
        self.radius = radius
        self.radius_floor = int(np.ceil(radius) - 1)
        r = int(radius)
        n_dst, n_groups = ctypes.c_int(), ctypes.c_int()
        glen = (ctypes.c_int * (4 * r))()
        gpaths = (ctypes.c_int * (4 * r))()
        _lib.check(L.irn_path_index_shape(r, ctypes.byref(n_dst), ctypes.byref(n_groups), glen, gpaths), "irn_path_index_shape")
        n_dst, n_groups = n_dst.value, n_groups.value
        Hp, Wp = int(default_size[0]), int(default_size[1])
        n_src = (Hp - self.radius_floor) * (Wp - 2 * self.radius_floor)
        n_pts = sum(glen[g] * gpaths[g] for g in range(n_groups))
        self.search_dst = np.empty((n_dst, 2), np.int64)
        paths = np.empty((n_pts, 2), np.int64)
        pidx = np.empty((n_pts, max(n_src, 0)), np.int64)
        self.src_indices = np.empty((max(n_src, 0),), np.int64)
        self.dst_indices = np.empty((n_dst, max(n_src, 0)), np.int64)
        _lib.check(L.irn_path_index_fill(r, Hp, Wp, self.search_dst.ctypes.data, paths.ctypes.data, pidx.ctypes.data,
                                         self.src_indices.ctypes.data, self.dst_indices.ctypes.data), "irn_path_index_fill")
        self.search_paths, self.path_indices = [], []
        o = 0
        for g in range(n_groups):
            n = glen[g] * gpaths[g]
            self.search_paths.append(paths[o:o + n].reshape(gpaths[g], glen[g], 2))
            self.path_indices.append(pidx[o:o + n].reshape(gpaths[g], glen[g], n_src))
            o += n


def stream_key(device):
    """Cache key of the work the caller is about to enqueue: (device index, current stream).  Device buffers cached under it are
    allocated on that stream and used only by work on that stream, so calls on two streams never share bytes, and dropping a
    buffer hands it back to the caching allocator in that stream's order, behind every call that used it (no record_stream)."""
    device = torch.device(device)
    return device.index, torch.cuda.current_stream(device).cuda_stream


_workspaces = {}


def _workspace(nbytes, device):
    """Scratch of at least `nbytes` for one call on the current stream of `device`, kept for the next call on that stream."""
    key = stream_key(device)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(int(nbytes * 1.25) + 256, dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


_scratches = {}


def _scratch(device):
    """rw_labels' global-max word, one per (device, stream) (see stream_key)."""
    key = stream_key(device)
    if key not in _scratches:
        _scratches[key] = torch.empty(256, dtype=torch.uint8, device=device)
    return _scratches[key]


def edge_to_affinity(edge, radius=5):
    """misc/indexing.py:91-109 on the un-padded grid.  edge cuda fp32 [B,h,w] (or [h,w]) ->
    [B, n_dst, h, w]; channel order = PathIndex.search_dst order."""
    _lib.require_cuda(edge)
    e = edge.reshape((-1,) + tuple(edge.shape[-2:])).contiguous().float()
    B, h, w = e.shape
    n_dst = ctypes.c_int()
    L = _lib.lib()
    _lib.check(L.irn_path_index_shape(int(radius), ctypes.byref(n_dst), None, None, None))
    out = torch.empty((B, n_dst.value, h, w), dtype=torch.float32, device=e.device)
    with torch.cuda.device(e.device):
        _lib.check(L.irn_edge_to_affinity(_lib.ptr(e), _lib.ptr(out), B, h, w, int(radius), _lib.stream_ptr()), "irn_edge_to_affinity")
    return out


class _ToAffinity(torch.autograd.Function):
    """Forward/backward pair behind `to_affinity`: one gather-max kernel that remembers where each maximum was, one scatter."""

    @staticmethod
    def forward(ctx, edge, radius):
        B, h, w = edge.shape
        rf = int(radius) - 1
        n_dst = ctypes.c_int()
        L = _lib.lib()
        _lib.check(L.irn_path_index_shape(int(radius), ctypes.byref(n_dst), None, None, None))
        n_src = (h - rf) * (w - 2 * rf)
        if h - rf <= 0 or w - 2 * rf <= 0:
            raise _lib.IrnError("to_affinity: grid %dx%d too small for radius %d" % (h, w, radius))
        e = edge.detach().contiguous().float()
        aff = torch.empty((B, n_dst.value, n_src), dtype=torch.float32, device=e.device)
        need_grad = edge.requires_grad
        arg = torch.empty((B, n_dst.value, n_src), dtype=torch.int32, device=e.device) if need_grad else None
        with torch.cuda.device(e.device):
            _lib.check(L.irn_to_affinity_forward(_lib.ptr(e), _lib.ptr(aff), _lib.ptr(arg) if need_grad else None, B, h, w, int(radius),
                                                 _lib.stream_ptr()), "irn_to_affinity_forward")
        ctx.shape, ctx.radius = (B, h, w), int(radius)
        if need_grad:
            ctx.save_for_backward(arg)
        return aff

    @staticmethod
    def backward(ctx, grad_aff):
        (arg,) = ctx.saved_tensors
        B, h, w = ctx.shape
        g = grad_aff.contiguous().float()
        grad_edge = torch.empty((B, h, w), dtype=torch.float32, device=g.device)
        with torch.cuda.device(g.device):
            _lib.check(_lib.lib().irn_to_affinity_backward(_lib.ptr(g), _lib.ptr(arg), _lib.ptr(grad_edge), B, h, w, ctx.radius,
                                                           _lib.stream_ptr()), "irn_to_affinity_backward")
        return grad_edge, None


def to_affinity(edge, path_index=None, radius=None):
    """Drop-in body for `AffinityDisplacementLoss.to_affinity` (net/resnet50_irn.py:162-175), differentiable: edge cuda fp32
    [B,1,H,W] (what train_irn passes: sigmoid(edge_out)) or [B,H,W]; returns aff [B, n_dst, (H-rf)*(W-2rf)] in
    PathIndex.search_dst order.  The reference gathers `edge.view(B,-1)` with PathIndex.path_indices built for default_size (H,W)
    and max-pools each path; here the radius is all that is needed (`path_index.radius`, or `radius=`)."""
    _lib.require_cuda(edge)
    if radius is None:
        if path_index is None:
            raise ValueError("to_affinity needs a PathIndex or a radius")
        radius = int(path_index.radius)
    if edge.dim() == 4:
        if edge.shape[1] != 1:
            raise ValueError("to_affinity expects one edge channel, got %s" % (tuple(edge.shape),))
        edge = edge[:, 0]
    if edge.dim() != 3:
        raise ValueError("to_affinity expects [B,1,H,W] or [B,H,W], got %s" % (tuple(edge.shape),))
    return _ToAffinity.apply(edge, int(radius))


def random_walk_batch(x, edge, chan_offsets, radius=5, beta=10, n_iter=256, variant=0):
    """Batched walk through the C ABI.  x cuda fp32 [total_channels,h,w]; edge cuda fp32
    [n_img,h,w]; chan_offsets: int sequence [n_img+1].  Returns fp32 [total_channels,h,w]."""
    _lib.require_cuda(x, edge)
    L = _lib.lib()
    x = x.contiguous().float()
    edge = edge.contiguous().float()
    n_img, h, w = edge.shape
    offs = np.ascontiguousarray(np.asarray(chan_offsets, dtype=np.int32))
    if offs.shape != (n_img + 1,) or int(offs[-1]) != x.shape[0]:
        raise _lib.IrnError("random_walk_batch: chan_offsets %s does not match n_img=%d / channels=%d" % (offs.shape, n_img, x.shape[0]))
    out = torch.empty_like(x)
    if x.shape[0] == 0:
        return out
    need = L.irn_rw_workspace_bytes(n_img, h, w, int(x.shape[0]), int(radius))
    if need == 0:
        raise _lib.IrnError("irn_rw_workspace_bytes rejected n_img=%d h=%d w=%d C=%d radius=%s" % (n_img, h, w, x.shape[0], radius))
    ws = _workspace(need, x.device)
    with torch.cuda.device(x.device):
        rc = L.irn_random_walk_variant(_lib.ptr(x), _lib.ptr(edge), _lib.ptr(out), n_img, offs.ctypes.data, h, w, int(radius),
                                       float(beta), int(n_iter), _lib.ptr(ws), ws.numel(), int(variant), _lib.stream_ptr())
    _lib.check(rc, "irn_random_walk")
    return out


def last_walk_was_fused():
    """True when the last walk on this thread ran as the fused cluster kernel (one launch for all steps)."""
    return bool(_lib.lib().irn_rw_last_was_fused())


def propagate_to_edge(x, edge, radius=5, beta=10, exp_times=8):
    """misc/indexing.py:141-167.  x: cuda fp32, any shape ending in (h,w); edge cuda fp32
    [1,h,w].  Returns [C,1,h,w] with C = prod(x.shape[:-2])."""
    h, w = x.shape[-2:]
    xs = x.reshape(-1, h, w)
    rw = random_walk_batch(xs, edge.reshape(1, h, w), [0, xs.shape[0]], radius, beta, 2 ** int(exp_times))
    return rw.view(-1, 1, h, w)


def rw_labels(rw, keys, size, bg_thres=0.25, want_index=False, want_scores=False, out=None):
    """step/make_sem_seg_labels.py:37,43-49.  rw cuda fp32 [C,1,h,w] or [C,h,w]; keys: int
    sequence of 0-based class ids (len C) or None; size=(H,W).  Returns (labels uint8 [H,W]
    cuda, index int32 [H,W] | None, scores fp32 [C,H,W] | None)."""
    _lib.require_cuda(rw)
    L = _lib.lib()
    h, w = rw.shape[-2:]
    r = rw.reshape(-1, h, w).contiguous().float()
    C = r.shape[0]
    H, W = int(size[0]), int(size[1])
    dev = r.device
    if out is not None and (tuple(out.shape) != (H, W) or out.dtype != torch.uint8 or not out.is_contiguous() or out.device != dev):
        raise _lib.IrnError("rw_labels: `out` must be a contiguous uint8 [H,W] tensor on the walk's device")
    labels = out if out is not None else torch.empty((H, W), dtype=torch.uint8, device=dev)
    index = torch.empty((H, W), dtype=torch.int32, device=dev) if want_index else None
    scores = torch.empty((C, H, W), dtype=torch.float32, device=dev) if want_scores else None
    kh = None
    if keys is not None:
        kh = np.ascontiguousarray(np.pad(np.asarray(keys, dtype=np.int64) + 1, (1, 0), mode="constant").astype(np.int32))
    scratch = _scratch(dev)
    with torch.cuda.device(dev):
        rc = L.irn_rw_labels(_lib.ptr(r), C, h, w, H, W, float(bg_thres), kh.ctypes.data if kh is not None else None, _lib.ptr(labels), _lib.ptr(index),
                             _lib.ptr(scores), _lib.ptr(scratch), _lib.stream_ptr())
    _lib.check(rc, "irn_rw_labels")
    return labels, index, scores


class ThresholdSweep:
    """The confusion matrices of many background thresholds in one pass over the scores (include/irn_b200.h, S1b).  Row j of
    confusion() is `step._voc_eval.confusion` of the label maps at thresholds[j]: eval_cam's padded argmax for add_cam, rw_labels'
    for add_walk.  The thresholds are rounded to float32 (the type of the background plane), sorted and deduplicated.  Each stream
    the adds run on accumulates into a histogram of its own (see stream_key); confusion() finalises and adds them up."""

    def __init__(self, thresholds, n_class, device):
        t = np.asarray(thresholds, dtype=np.float64).reshape(-1).astype(np.float32)
        if np.isnan(t).any():
            raise _lib.IrnError("ThresholdSweep: a threshold is NaN")
        self.thresholds = np.unique(t)
        self.n_class = int(n_class)
        self.device = torch.device(device)
        self._nbytes = _lib.lib().irn_threshold_sweep_bytes(len(self.thresholds), self.n_class)
        if self._nbytes == 0:
            raise _lib.IrnError("ThresholdSweep: %d distinct thresholds and %d classes (need 1..256 and 1..129)" %
                                (len(self.thresholds), self.n_class))
        self._acc = {}

    def _add(self, source, scores, C, h, w, keys, size, gt):
        H, W = int(size[0]), int(size[1])
        _lib.require_cuda(scores, gt)
        if scores.device != self.device or gt.device != self.device:
            raise _lib.IrnError("ThresholdSweep: inputs must be on %s" % self.device)
        if gt.dtype != torch.uint8 or tuple(gt.shape) != (H, W):
            raise _lib.IrnError("ThresholdSweep: ground truth must be uint8 [%d,%d], got %s %s" % (H, W, gt.dtype, tuple(gt.shape)))
        kh = np.ascontiguousarray(np.pad(np.asarray(keys, dtype=np.int64).reshape(-1) + 1, (1, 0)).astype(np.int32))
        if len(kh) != C + 1:
            raise _lib.IrnError("ThresholdSweep: %d keys for %d score planes" % (len(kh) - 1, C))
        key = stream_key(self.device)
        if key not in self._acc:
            self._acc[key] = (torch.cuda.current_stream(self.device), torch.zeros(self._nbytes, dtype=torch.uint8, device=self.device),
                              torch.empty(256, dtype=torch.uint8, device=self.device))
        _, hist, scratch = self._acc[key]
        g = gt.contiguous()
        with torch.cuda.device(self.device):
            rc = _lib.lib().irn_threshold_sweep_accumulate(source, _lib.ptr(scores), C, h, w, H, W, kh.ctypes.data, _lib.ptr(g),
                                                           self.thresholds.ctypes.data, len(self.thresholds), self.n_class, _lib.ptr(hist),
                                                           _lib.ptr(scratch), _lib.stream_ptr())
        _lib.check(rc, "irn_threshold_sweep_accumulate")

    def add_cam(self, high_res, keys, gt):
        """high_res cuda fp32 [K,H,W] (make_cam's full-resolution CAMs, K may be 0); keys: the K 0-based class ids; gt cuda uint8 [H,W]
        (255 = ignore)."""
        s = high_res.contiguous().float()
        if s.dim() != 3:
            raise _lib.IrnError("ThresholdSweep.add_cam: high_res must be [K,H,W], got %s" % (tuple(s.shape),))
        C, H, W = s.shape
        self._add(0, s, C, H, W, keys, (H, W), gt)

    def add_walk(self, rw, keys, size, gt):
        """rw cuda fp32 [C,1,h,w] or [C,h,w] (one image's walk, C may be 0); keys: the C 0-based class ids; size = (H,W); gt cuda uint8
        [H,W] (255 = ignore)."""
        h, w = rw.shape[-2:]
        r = rw.reshape(-1, h, w).contiguous().float()
        self._add(1, r, r.shape[0], h, w, keys, size, gt)

    def confusion(self):
        """int64 [T,n_class,n_class] over every image added so far: rows = ground truth, columns = prediction."""
        T, n = len(self.thresholds), self.n_class
        out = np.zeros((T, n, n), np.int64)
        for stream, hist, _ in self._acc.values():
            with torch.cuda.device(self.device), torch.cuda.stream(stream):
                conf = torch.empty((T, n, n), dtype=torch.int64, device=self.device)
                _lib.check(_lib.lib().irn_threshold_sweep_finalize(_lib.ptr(hist), T, n, _lib.ptr(conf), _lib.stream_ptr()),
                           "irn_threshold_sweep_finalize")
                out += conf.cpu().numpy()
        return out
