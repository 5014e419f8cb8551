"""Oracle (test infrastructure only): restatement of the per-image bodies of the three
label-generation steps.

 * cam_merge            step/make_cam.py:28-56
 * sem_seg_labels       step/make_sem_seg_labels.py:34-49
 * find_centroids       step/make_ins_seg_labels.py:18-56
 * cluster_centroids    step/make_ins_seg_labels.py:58-75 (+ misc/imutils.py:182-190,
                        misc/pyutils.py:86-101)
 * ins_seg_labels       step/make_ins_seg_labels.py:133-152 (+ detect_instance :82-105)
 * split_indices        misc/torchutils.py:66-68

Connected components use scipy.ndimage.label (4-connectivity) in place of
skimage.measure.label, which is absent here: "parity unpinned" for that one call.
"""
import numpy as np
import torch
import torch.nn.functional as F


def strided_size(size, stride):
    # misc/imutils.py:173-174
    return ((size[0] - 1) // stride + 1, (size[1] - 1) // stride + 1)


def cam_merge(outputs, size, label):
    """outputs: list of per-scale CAMs [20,hs,ws] (torch fp32); size=(H,W); label fp32[20].
    Returns keys int64[K], cam fp32 [K,ceil(H/4),ceil(W/4)], high_res fp32 [K,H,W]."""
    s4 = strided_size(size, 4)
    s16 = strided_size(size, 16)
    up = (s16[0] * 16, s16[1] * 16)
    low = sum(F.interpolate(o[None], s4, mode="bilinear", align_corners=False)[0] for o in outputs)
    high = sum(F.interpolate(o[:, None], up, mode="bilinear", align_corners=False) for o in outputs)
    high = high[:, 0, :size[0], :size[1]]
    keys = torch.nonzero(label)[:, 0]
    low = low[keys]
    low = low / (low.amax(dim=(1, 2), keepdim=True) + 1e-5)
    high = high[keys]
    high = high / (high.amax(dim=(1, 2), keepdim=True) + 1e-5)
    return keys, low, high


def upsample4_norm(rw, size):
    """x4 bilinear, crop to (H,W), divide by the global max
    (step/make_sem_seg_labels.py:43-44).  rw [C,1,h,w] -> [C,H,W]."""
    up = F.interpolate(rw, scale_factor=4, mode="bilinear", align_corners=False)[:, 0, :size[0], :size[1]]
    return up / torch.max(up)


def sem_seg_labels(rw, keys, size, bg_thres=0.25):
    """rw [K,1,h,w] torch fp32; keys int64[K] (0-based classes) -> uint8 [H,W]
    (step/make_sem_seg_labels.py:37,43-51)."""
    up = upsample4_norm(rw, size)
    bg = F.pad(up, (0, 0, 0, 0, 1, 0), value=bg_thres)
    pred = torch.argmax(bg, dim=0).numpy()
    k = np.pad(np.asarray(keys) + 1, (1, 0), mode="constant")
    return k[pred].astype(np.uint8)


def find_centroids(dp, iterations=300):
    """dp fp32 [2,h,w] -> int32 [2,h,w].  Expression order as written in the reference.
    NOTE numpy promotion: `centroid - floor(...).astype(int32)` is float32 - int32 = FLOAT64,
    so the bilinear update is evaluated in float64 (four products summed left to right, no
    FMA) and rounded to float32 only by the in-place `+=`; then clip, final round-half-even."""
    dp = np.asarray(dp, np.float32)
    h, w = dp.shape[1:]
    cy = np.repeat(np.arange(h, dtype=np.float32)[:, None], w, 1)
    cx = np.repeat(np.arange(w, dtype=np.float32)[None, :], h, 0)
    one = np.float32(1)
    for _ in range(iterations):
        uy = np.ceil(cy).astype(np.int32)
        ly = np.floor(cy).astype(np.int32)
        fy = cy - ly
        ux = np.ceil(cx).astype(np.int32)
        lx = np.floor(cx).astype(np.int32)
        fx = cx - lx
        step = []
        for c in (0, 1):
            f = dp[c]
            step.append(f[uy, ux] * fy * fx + f[ly, ux] * (one - fy) * fx
                        + f[uy, lx] * fy * (one - fx) + f[ly, lx] * (one - fy) * (one - fx))
        cy = np.clip((cy + step[0]).astype(np.float32), 0, h - 1)
        cx = np.clip((cx + step[1]).astype(np.float32), 0, w - 1)
    return np.stack([np.round(cy).astype(np.int32), np.round(cx).astype(np.int32)], 0)


def cc_label(mask):
    """4-connected components, background 0, raster-order numbering."""
    import scipy.ndimage as ndi
    return ndi.label(np.asarray(mask) != 0)[0]


def compress_range(arr):
    # misc/imutils.py:182-190
    u, inv = np.unique(arr, return_inverse=True)
    return inv.reshape(arr.shape).astype(np.int32)


def one_hot(a, n=None):
    # misc/pyutils.py:86-101
    a = np.asarray(a)
    n = int(a.max()) + 1 if n is None else n
    return (np.arange(n).reshape((n,) + (1,) * a.ndim) == a[None]).astype(bool)


def cluster_map(centroids, dp, thres=2.5):
    """cluster_centroids before its one_hot: int32 [h,w] instance ids in compress_range order (for cases with too many
    instances to hold the one-hot planes)."""
    strength = np.sqrt(dp[1] ** 2 + dp[0] ** 2)
    h, w = strength.shape
    lab = cc_label(strength < thres).reshape(-1)
    cl = lab[centroids[0] * w + centroids[1]].reshape(h, w)
    return compress_range(cl + 1)


def cluster_centroids(centroids, dp, thres=2.5):
    """-> bool [I,h,w] (step/make_ins_seg_labels.py:58-75)."""
    return one_hot(cluster_map(centroids, dp, thres))


def detect_instance(score_map, mask, class_id, max_fragment_size=0):
    """step/make_ins_seg_labels.py:82-105."""
    sc, lb, mk = [], [], []
    for s, m, c in zip(score_map, mask, class_id):
        if m.sum() < 1:
            continue
        for seg in one_hot(cc_label(m))[1:]:
            sc.append(0 if seg.sum() < max_fragment_size else np.max(s * seg))
            lb.append(c)
            mk.append(seg)
    return {"score": np.stack(sc, 0), "mask": np.stack(mk, 0), "class": np.stack(lb, 0)}


def ins_seg_labels(cams, keys, edge, dp, size, beta=10, exp_times=8, bg_thres=0.25, walk=None):
    """step/make_ins_seg_labels.py:131-150 for one image: centroids -> instance clusters -> per-instance seeds ->
    walk -> x4 up, /max, bg plane, argmax -> one-hot -> detect_instance.  cams fp32 [K,h,w], keys int64 [K], edge [1,h,w],
    dp [2,h,w] (numpy).  `walk(seeds[K*I,h,w], edge) -> [K*I,h,w]`; default = the exact fp64 stencil operator
    (the reference's dense fp32 squaring is its own 3-7e-5 away from it, SURVEY.md App. B)."""
    from . import indexing as oi
    dp = np.asarray(dp, np.float32)
    cen = find_centroids(dp)
    inst = cluster_centroids(cen, dp)                                           # bool [I,h,w]
    seeds = np.asarray(cams, np.float32)[:, None] * inst[None].astype(np.float32)   # :77-80  [K,I,h,w]
    K, I = seeds.shape[:2]
    flat = seeds.reshape(K * I, *seeds.shape[2:])
    if walk is None:
        rw = oi.propagate_stencil(flat, np.asarray(edge, np.float32), 5, beta, 2 ** exp_times).astype(np.float32)
    else:
        rw = walk(flat, edge)
    rw = torch.from_numpy(np.ascontiguousarray(rw, np.float32)).reshape(K * I, 1, *seeds.shape[2:])
    up = upsample4_norm(rw, size)
    bg = F.pad(up, (0, 0, 0, 0, 1, 0), value=bg_thres)
    shape = one_hot(torch.argmax(bg, 0).numpy(), K * I + 1)[1:]
    cls = np.repeat(np.asarray(keys), I)
    return detect_instance(up.numpy(), shape, cls, max_fragment_size=size[0] * size[1] * 0.01)


def split_indices(n_items, n_splits):
    # misc/torchutils.py:66-68
    return [np.arange(i, n_items, n_splits) for i in range(n_splits)]


def confusion_miou(preds, labels, n_class=21):
    """Confusion-matrix mIoU as in step/eval_sem_seg.py:18-31 (chainercv's
    calc_semantic_segmentation_confusion restated: rows = ground truth, cols = prediction,
    label 255/-1 ignored)."""
    conf = np.zeros((n_class, n_class), np.int64)
    for p, l in zip(preds, labels):
        p = np.asarray(p).reshape(-1).astype(np.int64)
        l = np.asarray(l).reshape(-1).astype(np.int64)
        ok = (l >= 0) & (l < n_class)
        conf += np.bincount(n_class * l[ok] + p[ok], minlength=n_class ** 2).reshape(n_class, n_class)
    gtj, resj, d = conf.sum(1), conf.sum(0), np.diag(conf)
    with np.errstate(divide="ignore", invalid="ignore"):
        iou = d / (gtj + resj - d)
    return iou, float(np.nanmean(iou))
