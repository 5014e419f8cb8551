"""Fully connected CRF on the device (N3): torch wrappers of irn_dense_crf / irn_ir_label (irn_b200/csrc/crf.cu).

The CRF is misc/imutils.py:156-170's (pydensecrf DenseCRF2D: a Gaussian and a bilateral Potts term, mean-field inference on the
permutohedral lattice) with the arithmetic oracle/crf.py states.  A batch holds images of one size; it is run in chunks so the
workspace (about 1.3 KB per pixel for 21 labels) stays under `max_workspace_bytes`."""
import ctypes

import numpy as np
import torch

from . import _lib

MAX_WORKSPACE_BYTES = 3 << 30


def max_labels():
    return int(_lib.lib().irn_crf_max_labels())


def _chunks(n, per_image_bytes, limit):
    step = max(1, min(n, int(limit // max(per_image_bytes, 1))))
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def _check_images(images_u8):
    _lib.require_cuda(images_u8)
    if images_u8.dtype != torch.uint8 or images_u8.dim() != 4 or images_u8.shape[-1] != 3:
        raise _lib.IrnError("images must be uint8 [n,H,W,3]; got %s %s" % (images_u8.dtype, tuple(images_u8.shape)))
    return images_u8.contiguous()


def dense_crf(images_u8, labels, n_labels, t=10, gt_prob=0.7, gauss=(3.0, 3.0), bilateral=(50.0, 5.0, 10.0), want_q=False,
              max_workspace_bytes=MAX_WORKSPACE_BYTES):
    """images_u8 uint8 [n,H,W,3], labels int [n,H,W] in [0, n_labels) (CUDA tensors) -> (labels int32 [n,H,W] = argmax of Q,
    Q fp32 [n,n_labels,H,W] or None, vertex counts int32 numpy [n,2] (Gaussian, bilateral lattice)).
    gauss = (sxy, compat), bilateral = (sxy, srgb, compat): addPairwiseGaussian / addPairwiseBilateral's arguments."""
    images_u8 = _check_images(images_u8)
    _lib.require_cuda(labels)
    n, H, W = images_u8.shape[:3]
    if tuple(labels.shape) != (n, H, W):
        raise _lib.IrnError("labels must be [n,H,W] = %s; got %s" % ((n, H, W), tuple(labels.shape)))
    n_labels = int(n_labels)
    if not 1 <= n_labels <= max_labels():
        raise _lib.IrnError("n_labels=%d outside [1, %d]" % (n_labels, max_labels()))
    L = _lib.lib()
    dev = images_u8.device
    labels = labels.to(torch.int32).contiguous()
    out = torch.empty((n, H, W), dtype=torch.int32, device=dev)
    q = torch.empty((n, n_labels, H, W), dtype=torch.float32, device=dev) if want_q else None
    counts = np.zeros((n, 2), np.int32)
    per_image = L.irn_crf_workspace_bytes(1, H, W, 1, n_labels)
    with torch.cuda.device(dev):
        for a, b in _chunks(n, per_image, max_workspace_bytes):
            nb = L.irn_crf_workspace_bytes(b - a, H, W, 1, n_labels)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            c = np.zeros((b - a, 2), np.int32)
            _lib.check(L.irn_dense_crf(_lib.ptr(images_u8[a:b]), _lib.ptr(labels[a:b]), b - a, H, W, n_labels, int(t), float(gt_prob),
                                       float(gauss[0]), float(gauss[1]), float(bilateral[0]), float(bilateral[1]), float(bilateral[2]),
                                       _lib.ptr(out[a:b]), _lib.ptr(q[a:b] if q is not None else None),
                                       c.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), nb, _lib.stream_ptr()), "irn_dense_crf")
            counts[a:b] = c
    return out, q, counts


def ir_labels(images_u8, high_res_list, keys_list, fg, bg, return_counts=False, max_workspace_bytes=MAX_WORKSPACE_BYTES):
    """step/cam_to_ir_label.py:19-41 for a batch of equally-sized images: images_u8 uint8 [n,H,W,3] (CUDA), high_res_list[i] fp32
    [K_i,H,W] (make_cam's `high_res`; host or device), keys_list[i] int [K_i] (make_cam's `keys`), fg / bg = conf_fg_thres /
    conf_bg_thres -> uint8 [n,H,W] conf maps (0 = background, 255 = unsure, else class + 1) on the images' device."""
    images_u8 = _check_images(images_u8)
    n, H, W = images_u8.shape[:3]
    if len(high_res_list) != n or len(keys_list) != n:
        raise _lib.IrnError("ir_labels: %d images, %d high_res, %d keys" % (n, len(high_res_list), len(keys_list)))
    L = _lib.lib()
    dev = images_u8.device
    keys = [np.asarray(k, np.int64).reshape(-1) for k in keys_list]
    counts = np.array([k.size for k in keys], np.int32)
    for i, h in enumerate(high_res_list):
        if tuple(h.shape) != (counts[i], H, W):
            raise _lib.IrnError("ir_labels: high_res %d has shape %s, want %s" % (i, tuple(h.shape), (int(counts[i]), H, W)))
    if counts.max(initial=0) + 1 > max_labels():
        raise _lib.IrnError("ir_labels: %d classes in one image (at most %d)" % (counts.max(), max_labels() - 1))
    planes = [torch.as_tensor(h, dtype=torch.float32) for h in high_res_list if h.shape[0] > 0]
    high = torch.cat([p.to(dev) for p in planes], 0).contiguous() if planes else None
    keys_all = np.ascontiguousarray(np.concatenate(keys + [np.zeros(0, np.int64)]).astype(np.int32))
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    out = torch.empty((n, H, W), dtype=torch.uint8, device=dev)
    vcounts = np.zeros((n, 2), np.int32)
    max_l = int(counts.max(initial=0)) + 1
    per_image = L.irn_crf_workspace_bytes(1, H, W, 2, max_l)
    with torch.cuda.device(dev):
        for a, b in _chunks(n, per_image, max_workspace_bytes):
            nb = L.irn_crf_workspace_bytes(b - a, H, W, 2, int(counts[a:b].max()) + 1)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            hi = high[offs[a]:offs[b]] if high is not None and offs[b] > offs[a] else None
            ck = np.ascontiguousarray(counts[a:b])
            kk = np.ascontiguousarray(keys_all[offs[a]:offs[b]]) if offs[b] > offs[a] else np.zeros(1, np.int32)
            c = np.zeros((b - a, 2), np.int32)
            _lib.check(L.irn_ir_label(_lib.ptr(images_u8[a:b]), _lib.ptr(hi), kk.ctypes.data_as(ctypes.c_void_p),
                                      ck.ctypes.data_as(ctypes.c_void_p), b - a, H, W, float(fg), float(bg), _lib.ptr(out[a:b]),
                                      c.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), nb, _lib.stream_ptr()), "irn_ir_label")
            vcounts[a:b] = c
    return (out, vcounts) if return_counts else out


def set_timing(enable):
    _lib.check(_lib.lib().irn_crf_set_timing(int(bool(enable))), "irn_crf_set_timing")


def last_ms():
    """(lattice build, iterations, tail) device milliseconds of the last timed call on this thread."""
    ms = (ctypes.c_float * 3)()
    _lib.check(_lib.lib().irn_crf_last_ms(ms), "irn_crf_last_ms")
    return tuple(float(x) for x in ms)
