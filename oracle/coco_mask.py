"""Numpy oracle of irn_b200/csrc/coco_mask.cu: COCO ground-truth rasterisation, the bit-plane layout, and mask overlap counts.

Polygons (pycocotools' rleFrPoly, restated from its published algorithm; pycocotools itself is not pinned here):
  1. vertices upsampled x5 and truncated toward zero: (int)(5*v + .5), the polygon closed by repeating vertex 0;
  2. every edge walked along its major axis from its start to its end, one sample per unit step: with dx = |xe-xs|, dy = |ye-ys|, the
     edge is flipped when (dx >= dy and xs > xe) or (dx < dy and ys > ye), slope s = (ye-ys)/dx (or (xe-xs)/dy), sample t at
     (xs+t, (int)(ys + s*t + .5)) (or ((int)(xs + s*t + .5), ys+t)), t running dx..0 for a flipped edge so the samples always go from
     the original start to the original end; the samples of all edges are concatenated (a zero-length edge's 0/0 slope gives the
     x86 conversion of NaN, INT_MIN, as its row);
  3. for each pair of consecutive samples whose x differs: column xd = (min(u) if x decreased else u-1) mapped back as (xd+.5)/5-.5,
     skipped unless integral and within [0, w-1]; row yd = min of the two v, mapped back the same way, clamped to [0, h] and ceil'd;
  4. a pixel (x, y) is inside when the number of toggles (xd, yd) at or before column-major position x*h + y is odd (equal toggles
     cancel, as the zero-run merge of the C code does; a toggle at h*w is past the image).
  Every double operation is one IEEE operation in the order written (numpy ufuncs do not contract to fused multiply-adds).  A polygon
  of fewer than 3 vertices walks out and back over the same samples, so its toggles cancel: it is empty.  An annotation of several
  polygons is their union.
Uncompressed RLE ({"counts": [...], "size": [h, w]}): column-major runs starting with zeros.  Any other segmentation raises ValueError
naming the annotation id.

Bit plane of an h x w mask: w columns of ceil(h/32) uint32 words, bit b of word j of column x = pixel (32j+b, x), padding bits zero.
"""
import numpy as np

INT_MIN = -(1 << 31)


def _up5(v):
    return (np.float64(5.0) * np.asarray(v, np.float64) + 0.5).astype(np.int64)


def _edge_samples(xs, ys, xe, ye):
    dx, dy = abs(xe - xs), abs(ys - ye)
    flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
    if flip:
        xs, xe, ys, ye = xe, xs, ye, ys
    if dx >= dy:
        t = np.arange(dx + 1, dtype=np.int64)
        t = dx - t if flip else t
        if dx == 0:
            return t + xs, np.full(1, INT_MIN, np.int64)
        s = np.float64(ye - ys) / np.float64(dx)
        return t + xs, (np.float64(ys) + s * t.astype(np.float64) + 0.5).astype(np.int64)
    t = np.arange(dy + 1, dtype=np.int64)
    t = dy - t if flip else t
    s = np.float64(xe - xs) / np.float64(dy)
    return (np.float64(xs) + s * t.astype(np.float64) + 0.5).astype(np.int64), t + ys


def poly_toggles(xy, h, w):
    """Flat column-major toggle positions (x*h + y, y in [0, h]) of one polygon, xy float64 [2k] as in the JSON."""
    xy = np.asarray(xy, np.float64).reshape(-1)
    k = len(xy) // 2
    if k == 0:
        return np.zeros(0, np.int64)
    x, y = _up5(xy[0:2 * k:2]), _up5(xy[1:2 * k:2])
    x, y = np.append(x, x[0]), np.append(y, y[0])
    us, vs = [], []
    for j in range(k):
        u, v = _edge_samples(int(x[j]), int(y[j]), int(x[j + 1]), int(y[j + 1]))
        us.append(u)
        vs.append(v)
    u, v = np.concatenate(us), np.concatenate(vs)
    ch = np.flatnonzero(u[1:] != u[:-1]) + 1
    xd = np.where(u[ch] < u[ch - 1], u[ch], u[ch] - 1).astype(np.float64)
    xd = (xd + 0.5) / 5.0 - 0.5
    yd = np.minimum(v[ch], v[ch - 1]).astype(np.float64)
    yd = np.ceil(np.clip((yd + 0.5) / 5.0 - 0.5, 0.0, float(h)))
    ok = (np.floor(xd) == xd) & (xd >= 0) & (xd <= w - 1)
    return xd[ok].astype(np.int64) * h + yd[ok].astype(np.int64)


def toggles_to_mask(pos, h, w):
    """bool [h,w]: pixels with an odd number of toggles at or before their column-major position."""
    pos = np.asarray(pos, np.int64)
    pos = pos[pos < h * w]
    t = np.bincount(pos, minlength=h * w) & 1
    inside = (np.cumsum(t) & 1).astype(bool)
    return inside.reshape(w, h).T.copy()


def rle_decode(rle):
    h, w = (int(s) for s in rle["size"])
    counts = np.asarray(rle["counts"], np.int64)
    if counts.sum() != h * w:
        raise ValueError("RLE counts add up to %d, size %dx%d" % (counts.sum(), h, w))
    return toggles_to_mask(np.cumsum(counts)[:-1] if len(counts) else np.zeros(0, np.int64), h, w)


def ann_mask(segm, h, w, ann_id=None):
    """bool [h,w] of one annotation's segmentation (polygon list or uncompressed RLE)."""
    if isinstance(segm, list):
        m = np.zeros((h, w), bool)
        for p in segm:
            m |= toggles_to_mask(poly_toggles(p, h, w), h, w)
        return m
    if isinstance(segm, dict) and isinstance(segm.get("counts"), list):
        if [int(s) for s in segm["size"]] != [h, w]:
            raise ValueError("annotation %s: RLE size %s, image %dx%d" % (ann_id, segm["size"], h, w))
        return rle_decode(segm)
    raise ValueError("annotation %s: unsupported segmentation (polygons or uncompressed RLE only)" % ann_id)


def pack(mask):
    """bool [h,w] -> uint32 [w * ceil(h/32)] in the bit-plane layout."""
    mask = np.asarray(mask, bool)
    h, w = mask.shape
    cw = (h + 31) // 32
    col = np.zeros((w, cw * 32), bool)
    col[:, :h] = mask.T
    bits = col.reshape(w, cw, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)
    return bits.sum(axis=2).astype(np.uint32).reshape(-1)


def overlaps(pred, gt):
    """pred bool [M,h,w], gt bool [G,h,w] -> (inter int64 [M,G], area_pred int64 [M], area_gt int64 [G])."""
    pred, gt = np.asarray(pred, bool), np.asarray(gt, bool)
    p = pred.reshape(len(pred), int(np.prod(pred.shape[1:]))).astype(np.int64)
    g = gt.reshape(len(gt), int(np.prod(gt.shape[1:]))).astype(np.int64)
    return p @ g.T, p.sum(1), g.sum(1)
