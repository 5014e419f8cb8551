"""The slice of the reference's ``misc/imutils.py`` the label-generation steps use."""
import numpy as np
from PIL import Image


def pil_resize(img, size, order):
    """misc/imutils.py:8-17 -- PIL BICUBIC (order 3) / NEAREST (order 0) to size=(h, w)."""
    if size[0] == img.shape[0] and size[1] == img.shape[1]:
        return img
    resample = {3: Image.BICUBIC, 0: Image.NEAREST}[order]
    return np.asarray(Image.fromarray(img).resize(size[::-1], resample))


def pil_rescale(img, scale, order):
    """misc/imutils.py:19-22."""
    h, w = img.shape[:2]
    return pil_resize(img, (int(np.round(h * scale)), int(np.round(w * scale))), order)


def get_strided_size(orig_size, stride):
    """misc/imutils.py:173-174."""
    return ((orig_size[0] - 1) // stride + 1, (orig_size[1] - 1) // stride + 1)


def get_strided_up_size(orig_size, stride):
    """misc/imutils.py:177-179."""
    s = get_strided_size(orig_size, stride)
    return s[0] * stride, s[1] * stride


def compress_range(arr):
    """misc/imutils.py:182-190: relabel the distinct values of arr as 0..n-1 in ascending order."""
    _, inv = np.unique(arr, return_inverse=True)
    return inv.reshape(arr.shape).astype(np.int32)


def HWC_to_CHW(img):
    return np.transpose(img, (2, 0, 1))


def crf_inference_label(img, labels, t=10, n_labels=21, gt_prob=0.7):
    """misc/imutils.py:156-170: the dense CRF (Gaussian sxy=3 compat=3, bilateral sxy=50 srgb=5 compat=10, t mean-field
    iterations) of uint8 [H,W,3] `img` with the unary of the label map `labels` [H,W], argmax over labels.  numpy in, numpy out
    (int64 [H,W]); computed on the current CUDA device (irn_b200.crf).  n_labels == 1 gives label 0 everywhere."""
    import torch
    from .. import crf
    dev = torch.device("cuda", torch.cuda.current_device())
    x = torch.from_numpy(np.ascontiguousarray(img, dtype=np.uint8))[None].to(dev)
    lab = torch.from_numpy(np.ascontiguousarray(labels, dtype=np.int32))[None].to(dev)
    out, _, _ = crf.dense_crf(x, lab, n_labels, t=t, gt_prob=gt_prob)
    return out[0].cpu().numpy().astype(np.int64)
