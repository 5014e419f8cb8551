"""The background-threshold sweep restated in numpy: the confusion matrices of step/eval_cam.py:15-18 (and of
step/make_sem_seg_labels.py:43-49 + step/eval_sem_seg.py, given the normalised walk) at T thresholds from one pass over the scores.

At threshold t, argmax over [t, s_0, .., s_{K-1}] is the foreground argmax c (np.argmax: first maximum, first NaN) when its value m
exceeds t, else 0 (background).  c and m do not depend on t: each pixel is binned by (ground truth g, keys[c]+1, b = number of
thresholds below m; T for NaN), and threshold j's confusion is the suffix sum over b > j, its background column the rest of row g."""
import numpy as np


def sweep_confusion(scores, keys, gts, thresholds, n_class):
    """scores: list of fp32 [K,H,W] (K may be 0); keys: list of the K 0-based class ids; gts: list of int [H,W], -1 = ignore;
    thresholds: strictly ascending float32 [T].  Returns int64 [T,n_class,n_class], rows = ground truth."""
    thr = np.asarray(thresholds, np.float32)
    T = len(thr)
    hist = np.zeros((n_class, n_class, T + 1), np.int64)
    for s, k, g in zip(scores, keys, gts):
        g = np.asarray(g).reshape(-1).astype(np.int64)
        ok = g >= 0
        s = np.asarray(s, np.float32)
        if s.shape[0] == 0:
            b = np.zeros(g.shape, np.int64)
            p = np.zeros(g.shape, np.int64)
        else:
            c = np.argmax(s, axis=0)
            m = np.take_along_axis(s, c[None], 0)[0].reshape(-1)
            b = np.searchsorted(thr, m, side="left").astype(np.int64)
            b[np.isnan(m)] = T
            p = (np.asarray(k, np.int64).reshape(-1) + 1)[c.reshape(-1)]
            p[b == 0] = 0
        g, p, b = g[ok], p[ok], b[ok]
        if (g >= n_class).any() or (p >= n_class).any():
            raise ValueError("label outside [0, %d)" % n_class)
        hist += np.bincount((g * n_class + p) * (T + 1) + b, minlength=hist.size).reshape(hist.shape)
    suffix = np.cumsum(hist[..., ::-1], axis=-1)[..., ::-1]          # suffix[g, p, b] = sum over b' >= b
    conf = np.ascontiguousarray(np.moveaxis(suffix[..., 1:], -1, 0))  # conf[j] = suffix at b = j + 1
    conf[:, :, 0] = hist.sum(axis=(1, 2))[None, :] - conf[:, :, 1:].sum(-1)
    return conf
