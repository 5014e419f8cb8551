"""Fully connected CRF on the device (N3): torch wrappers of irn_dense_crf / irn_ir_label (irn_b200/csrc/crf.cu).

The CRF is misc/imutils.py:156-170's (pydensecrf DenseCRF2D: a Gaussian and a bilateral Potts term, mean-field inference on the
permutohedral lattice) with the arithmetic oracle/crf.py states.  `dense_crf` / `ir_labels` take a batch of images of one size
([n,H,W,3]); `dense_crf_ragged` / `ir_labels_ragged` take images of any sizes packed back to back in one flat uint8 buffer (the
layout StepContext.pack_images and the exact JPEG decoder produce) and return their results packed the same way (`unpack` splits
them).  Image i's result is bit for bit the same either way, and whatever else is in its batch.  A batch is run in chunks so the
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


def _ragged_chunks(per_image, limit):
    """Consecutive [a, b) ranges whose per-image workspaces add up to at most `limit` (at least one image each)."""
    out, a, acc = [], 0, 0
    for i, nb in enumerate(per_image):
        if i > a and acc + nb > limit:
            out.append((a, i))
            a, acc = i, 0
        acc += nb
    out.append((a, len(per_image)))
    return out


def _check_flat(flat_u8, sizes):
    """-> (sizes as a list of (H, W), HOST int32 [n][2], pixel offsets int64 [n+1])."""
    _lib.require_cuda(flat_u8)
    if flat_u8.dtype != torch.uint8 or flat_u8.dim() != 1:
        raise _lib.IrnError("images must be one flat uint8 buffer; got %s %s" % (flat_u8.dtype, tuple(flat_u8.shape)))
    sizes = [(int(h), int(w)) for h, w in sizes]
    if not sizes or any(h <= 0 or w <= 0 for h, w in sizes):
        raise _lib.IrnError("bad image sizes %s" % (sizes,))
    offs = np.concatenate([[0], np.cumsum([h * w for h, w in sizes])]).astype(np.int64)
    if flat_u8.numel() != 3 * offs[-1]:
        raise _lib.IrnError("images: %d bytes, the sizes add up to %d" % (flat_u8.numel(), 3 * offs[-1]))
    return sizes, np.ascontiguousarray(np.asarray(sizes, np.int32).reshape(-1, 2)), offs


def unpack(flat, sizes, channels=None):
    """A packed per-image result -> list of views: [H_i,W_i] per image, or [channels,H_i,W_i] (dense_crf_ragged's Q)."""
    c = 1 if channels is None else int(channels)
    out, o = [], 0
    for h, w in sizes:
        v = flat[o:o + c * h * w]
        out.append(v.view(h, w) if channels is None else v.view(c, h, w))
        o += c * h * w
    return out


def dense_crf_ragged(flat_u8, sizes, labels, n_labels, t=10, gt_prob=0.7, gauss=(3.0, 3.0), bilateral=(50.0, 5.0, 10.0), want_q=False,
                     max_workspace_bytes=MAX_WORKSPACE_BYTES):
    """dense_crf for images of any sizes: flat_u8 uint8 [sum 3*H_i*W_i] (image i's [H_i,W_i,3] bytes back to back), sizes [(H_i, W_i)],
    labels int [sum H_i*W_i] (CUDA) -> (labels int32 [sum H_i*W_i], Q fp32 [n_labels * sum H_i*W_i] (image i's [n_labels,H_i,W_i] back
    to back) or None, vertex counts int32 numpy [n,2]); `unpack` splits the packed results."""
    sizes, hw, offs = _check_flat(flat_u8, sizes)
    _lib.require_cuda(labels)
    if labels.dim() != 1 or labels.numel() != offs[-1]:
        raise _lib.IrnError("labels must be flat [%d]; got %s" % (offs[-1], tuple(labels.shape)))
    n_labels = int(n_labels)
    if not 1 <= n_labels <= max_labels():
        raise _lib.IrnError("n_labels=%d outside [1, %d]" % (n_labels, max_labels()))
    L = _lib.lib()
    dev = flat_u8.device
    labels = labels.to(torch.int32).contiguous()
    n = len(sizes)
    out = torch.empty(int(offs[-1]), dtype=torch.int32, device=dev)
    q = torch.empty(n_labels * int(offs[-1]), dtype=torch.float32, device=dev) if want_q else None
    counts = np.zeros((n, 2), np.int32)
    per_image = [L.irn_crf_ragged_workspace_bytes(1, hw[i:i + 1].ctypes.data_as(ctypes.c_void_p), 1, n_labels) for i in range(n)]
    with torch.cuda.device(dev):
        for a, b in _ragged_chunks(per_image, max_workspace_bytes):
            s = np.ascontiguousarray(hw[a:b])
            nb = L.irn_crf_ragged_workspace_bytes(b - a, s.ctypes.data_as(ctypes.c_void_p), 1, n_labels)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            c = np.zeros((b - a, 2), np.int32)
            p0, p1 = int(offs[a]), int(offs[b])
            _lib.check(L.irn_dense_crf_ragged(_lib.ptr(flat_u8[3 * p0:3 * p1]), 3 * (p1 - p0), s.ctypes.data_as(ctypes.c_void_p), b - a,
                                              _lib.ptr(labels[p0:p1]), n_labels, int(t), float(gt_prob), float(gauss[0]), float(gauss[1]),
                                              float(bilateral[0]), float(bilateral[1]), float(bilateral[2]), _lib.ptr(out[p0:p1]),
                                              _lib.ptr(q[n_labels * p0:n_labels * p1] if q is not None else None),
                                              c.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), nb, _lib.stream_ptr()), "irn_dense_crf_ragged")
            counts[a:b] = c
    return out, q, counts


def _conf_inputs(what, sizes, high_res_list, keys_list, n_classes, dev):
    """The checks of the step's inputs -> (keys int32 [sum K_i], counts int32 [n], high_res planes flat on dev or None, element offset
    of each image's planes int64 [n+1])."""
    n = len(sizes)
    if len(high_res_list) != n or len(keys_list) != n:
        raise _lib.IrnError("%s: %d images, %d high_res, %d keys" % (what, n, len(high_res_list), len(keys_list)))
    keys = [np.asarray(k, np.int64).reshape(-1) for k in keys_list]
    counts = np.array([k.size for k in keys], np.int32)
    for i, h in enumerate(high_res_list):
        if tuple(h.shape) != (counts[i],) + tuple(sizes[i]):
            raise _lib.IrnError("%s: high_res %d has shape %s, want %s" % (what, i, tuple(h.shape), (int(counts[i]),) + tuple(sizes[i])))
    if not 1 <= int(n_classes) <= max_labels() - 1:
        raise _lib.IrnError("%s: n_classes=%s outside [1, %d]" % (what, n_classes, max_labels() - 1))
    if counts.max(initial=0) > n_classes:
        raise _lib.IrnError("%s: %d classes in one image (the dataset has %d)" % (what, counts.max(), n_classes))
    for i, k in enumerate(keys):
        if k.size and (k.min() < 0 or k.max() >= n_classes):
            raise _lib.IrnError("%s: image %d has class id %d outside [0, %d)" % (what, i, k.max() if k.max() >= n_classes else k.min(),
                                                                                  n_classes))
    planes = [torch.as_tensor(h, dtype=torch.float32) for h in high_res_list if h.shape[0] > 0]
    high = torch.cat([p.to(dev).reshape(-1) for p in planes], 0).contiguous() if planes else None
    keys_all = np.ascontiguousarray(np.concatenate(keys + [np.zeros(0, np.int64)]).astype(np.int32))
    elems = np.concatenate([[0], np.cumsum([int(c) * h * w for c, (h, w) in zip(counts, sizes)])]).astype(np.int64)
    return keys_all, counts, high, elems


def ir_labels(images_u8, high_res_list, keys_list, fg, bg, return_counts=False, max_workspace_bytes=MAX_WORKSPACE_BYTES, n_classes=20):
    """step/cam_to_ir_label.py:19-41 for a batch of equally-sized images: images_u8 uint8 [n,H,W,3] (CUDA), high_res_list[i] fp32
    [K_i,H,W] (make_cam's `high_res`; host or device), keys_list[i] int [K_i] (make_cam's `keys`), fg / bg = conf_fg_thres /
    conf_bg_thres -> uint8 [n,H,W] conf maps (0 = background, 255 = unsure, else class + 1) on the images' device.
    n_classes: the dataset's class count (20 PASCAL VOC, 80 MS COCO; at most max_labels() - 1): every key must be a class id in
    [0, n_classes), so an image has at most n_classes classes."""
    images_u8 = _check_images(images_u8)
    n, H, W = images_u8.shape[:3]
    L = _lib.lib()
    dev = images_u8.device
    keys_all, counts, high, elems = _conf_inputs("ir_labels", [(H, W)] * n, high_res_list, keys_list, n_classes, dev)
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    out = torch.empty((n, H, W), dtype=torch.uint8, device=dev)
    vcounts = np.zeros((n, 2), np.int32)
    max_l = int(counts.max(initial=0)) + 1
    per_image = L.irn_crf_workspace_bytes(1, H, W, 2, max_l)
    with torch.cuda.device(dev):
        for a, b in _chunks(n, per_image, max_workspace_bytes):
            nb = L.irn_crf_workspace_bytes(b - a, H, W, 2, int(counts[a:b].max()) + 1)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            hi = high[elems[a]:elems[b]] if high is not None and elems[b] > elems[a] else None
            ck = np.ascontiguousarray(counts[a:b])
            kk = np.ascontiguousarray(keys_all[offs[a]:offs[b]]) if offs[b] > offs[a] else np.zeros(1, np.int32)
            c = np.zeros((b - a, 2), np.int32)
            _lib.check(L.irn_ir_label(_lib.ptr(images_u8[a:b]), _lib.ptr(hi), kk.ctypes.data_as(ctypes.c_void_p),
                                      ck.ctypes.data_as(ctypes.c_void_p), b - a, H, W, float(fg), float(bg), _lib.ptr(out[a:b]),
                                      c.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), nb, _lib.stream_ptr()), "irn_ir_label")
            vcounts[a:b] = c
    return (out, vcounts) if return_counts else out


def ir_labels_ragged(flat_u8, sizes, high_res_list, keys_list, fg, bg, return_counts=False, max_workspace_bytes=MAX_WORKSPACE_BYTES,
                     n_classes=20):
    """ir_labels for images of any sizes: flat_u8 uint8 [sum 3*H_i*W_i] (CUDA; image i's [H_i,W_i,3] bytes back to back, as
    StepContext.pack_images returns them), sizes [(H_i, W_i)], high_res_list[i] fp32 [K_i,H_i,W_i], keys_list[i] int [K_i] ->
    uint8 [sum H_i*W_i]: image i's conf map [H_i,W_i] after images 0..i-1 (`unpack(out, sizes)` splits them); image i's bits are
    ir_labels' for that image alone."""
    sizes, hw, poffs = _check_flat(flat_u8, sizes)
    n = len(sizes)
    L = _lib.lib()
    dev = flat_u8.device
    keys_all, counts, high, elems = _conf_inputs("ir_labels_ragged", sizes, high_res_list, keys_list, n_classes, dev)
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    out = torch.empty(int(poffs[-1]), dtype=torch.uint8, device=dev)
    vcounts = np.zeros((n, 2), np.int32)
    max_l = int(counts.max(initial=0)) + 1
    per_image = [L.irn_crf_ragged_workspace_bytes(1, hw[i:i + 1].ctypes.data_as(ctypes.c_void_p), 2, max_l) for i in range(n)]
    with torch.cuda.device(dev):
        for a, b in _ragged_chunks(per_image, max_workspace_bytes):
            s = np.ascontiguousarray(hw[a:b])
            nb = L.irn_crf_ragged_workspace_bytes(b - a, s.ctypes.data_as(ctypes.c_void_p), 2, int(counts[a:b].max()) + 1)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            hi = high[elems[a]:elems[b]] if high is not None and elems[b] > elems[a] else None
            ck = np.ascontiguousarray(counts[a:b])
            kk = np.ascontiguousarray(keys_all[offs[a]:offs[b]]) if offs[b] > offs[a] else np.zeros(1, np.int32)
            c = np.zeros((b - a, 2), np.int32)
            p0, p1 = int(poffs[a]), int(poffs[b])
            _lib.check(L.irn_ir_label_ragged(_lib.ptr(flat_u8[3 * p0:3 * p1]), 3 * (p1 - p0), s.ctypes.data_as(ctypes.c_void_p), b - a,
                                             _lib.ptr(hi), int(elems[b] - elems[a]), kk.ctypes.data_as(ctypes.c_void_p),
                                             ck.ctypes.data_as(ctypes.c_void_p), float(fg), float(bg), _lib.ptr(out[p0:p1]),
                                             c.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), nb, _lib.stream_ptr()), "irn_ir_label_ragged")
            vcounts[a:b] = c
    return (out, vcounts) if return_counts else out


def set_timing(enable):
    _lib.check(_lib.lib().irn_crf_set_timing(int(bool(enable))), "irn_crf_set_timing")


def last_ms():
    """(lattice build, iterations, tail) device milliseconds of the last timed call on this thread."""
    ms = (ctypes.c_float * 3)()
    _lib.check(_lib.lib().irn_crf_last_ms(ms), "irn_crf_last_ms")
    return tuple(float(x) for x in ms)
