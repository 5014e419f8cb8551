"""The published COCO ``segm`` evaluation (pycocotools' COCOeval: evaluate, accumulate, summarize) restated in numpy, on exact integer
mask counts (irn_b200.coco.mask.overlaps).  pycocotools is not pinned here: agreement with it is not verified.

Parameters
  IoU thresholds   np.linspace(.5, .95, 10) (so the ninth is 0.8999999999999999)
  recall thresholds np.linspace(0, 1, 101)
  maxDets          1, 10, 100
  area ranges      all [0, 1e10], small [0, 32**2], medium [32**2, 96**2], large [96**2, 1e10]; an area a is outside [lo, hi] when
                   a < lo or a > hi (both bounds belong to the range)

IoU of detection d and ground truth g, float64 from the counts: 0 where they do not intersect, else inter / (area_d + area_g - inter),
or inter / area_d when g is a crowd region.

Per (image, category, area range), with maxDet = 100:
  - a ground truth is ignored when it is crowd or its JSON ``area`` lies outside the range; the ignored ones are moved after the others
    by a stable sort, so each group keeps its annotation order;
  - detections are sorted by descending score with a stable mergesort and cut to maxDet;
  - for each IoU threshold t, each detection in that order takes the best ground truth by scanning them in the sorted order with the
    bar min(t, 1 - 1e-10): a ground truth already matched at this threshold is skipped unless it is a crowd region (crowds can be
    matched again); the scan stops at the first ignored ground truth once a non-ignored one is held; a ground truth whose IoU is below
    the bar is skipped, otherwise it is held and the bar rises to its IoU, so on equal IoU the later ground truth wins;
  - a detection matched to an ignored ground truth is ignored; an unmatched detection is ignored when its mask area (the popcount)
    lies outside the range;
  - an (image, category) with neither ground truth nor detections takes no part.
Accumulate, per category, area range and maxDets m:
  - images in ascending COCO image id; each image's first m detections (in its score order) are concatenated in that order and sorted
    by descending score with a stable mergesort;
  - tp / fp = matched / unmatched detections that are not ignored, cumulated; recall = tp / (non-ignored ground truths); precision
    = tp / (tp + fp + np.spacing(1)); a category without non-ignored ground truth keeps -1;
  - precision is made monotone from the right (p[i-1] = max(p[i-1], p[i])), sampled at np.searchsorted(recall, recThrs,
    side="left"), 0 past the last recall; the recall entry is the final recall (0 with no detection).
Summarize: the 12 standard numbers (AP, AP50, AP75, AP small/medium/large at 100 detections; AR at 1, 10, 100; AR small/medium/large at
100): the mean over the entries > -1, or -1 when there is none.
"""
import numpy as np

IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = (1, 10, 100)
AREA_RNG = ((0, 1e5 ** 2), (0, 32 ** 2), (32 ** 2, 96 ** 2), (96 ** 2, 1e5 ** 2))
AREA_LBL = ("all", "small", "medium", "large")
STAT_NAMES = ("AP", "AP50", "AP75", "APs", "APm", "APl", "AR1", "AR10", "AR100", "ARs", "ARm", "ARl")


class ImageEval:
    """One image's inputs: ground truth (category index int [G], JSON area float [G] (selects the area range), crowd bool [G], pixel
    count int [G] (enters the IoU)), detections (category index int [D], score float [D], pixel count int [D]) and the intersection
    counts inter int [D,G]."""

    def __init__(self, image_id, gt_cat, gt_area, gt_crowd, gt_mask_area, dt_cat, dt_score, dt_area, inter):
        self.image_id = int(image_id)
        self.gt_cat = np.asarray(gt_cat, np.int64).reshape(-1)
        self.gt_area = np.asarray(gt_area, np.float64).reshape(-1)
        self.gt_crowd = np.asarray(gt_crowd, bool).reshape(-1)
        self.gt_mask_area = np.asarray(gt_mask_area, np.int64).reshape(-1)
        self.dt_cat = np.asarray(dt_cat, np.int64).reshape(-1)
        self.dt_score = np.asarray(dt_score, np.float64).reshape(-1)
        self.dt_area = np.asarray(dt_area, np.int64).reshape(-1)
        self.inter = np.asarray(inter, np.int64).reshape(len(self.dt_cat), len(self.gt_cat))


def iou(inter, area_d, area_g, crowd):
    inter = np.asarray(inter, np.float64)
    area_d = np.asarray(area_d, np.float64)[:, None]
    area_g = np.asarray(area_g, np.float64)[None, :]
    union = np.where(np.asarray(crowd, bool)[None, :], area_d, area_d + area_g - inter)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(inter > 0, inter / np.where(union > 0, union, 1.0), 0.0)


def evaluate_img(im, k, a_rng, max_det=MAX_DETS[-1]):
    """-> None, or dict(dt_scores [D'], dt_matched bool [T,D'], dt_ignore bool [T,D'], gt_ignore bool [G'])."""
    g_sel = np.flatnonzero(im.gt_cat == k)
    d_sel = np.flatnonzero(im.dt_cat == k)
    if len(g_sel) == 0 and len(d_sel) == 0:
        return None
    g_ig = im.gt_crowd[g_sel] | (im.gt_area[g_sel] < a_rng[0]) | (im.gt_area[g_sel] > a_rng[1])
    g_order = np.argsort(g_ig.astype(np.int64), kind="mergesort")
    g_sel, g_ig = g_sel[g_order], g_ig[g_order]
    crowd = im.gt_crowd[g_sel]
    d_order = np.argsort(-im.dt_score[d_sel], kind="mergesort")
    d_sel = d_sel[d_order][:max_det]
    ious = iou(im.inter[np.ix_(d_sel, g_sel)], im.dt_area[d_sel], im.gt_mask_area[g_sel], crowd)
    T, G, D = len(IOU_THRS), len(g_sel), len(d_sel)
    gtm = np.zeros((T, G), bool)
    dtm = np.zeros((T, D), bool)
    dt_ig = np.zeros((T, D), bool)
    if D and G:
        for ti, t in enumerate(IOU_THRS):
            for di in range(D):
                bar, m = min(t, 1 - 1e-10), -1
                for gi in range(G):
                    if gtm[ti, gi] and not crowd[gi]:
                        continue
                    if m > -1 and not g_ig[m] and g_ig[gi]:
                        break
                    if ious[di, gi] < bar:
                        continue
                    bar, m = ious[di, gi], gi
                if m == -1:
                    continue
                dt_ig[ti, di] = g_ig[m]
                dtm[ti, di] = True
                gtm[ti, m] = True
    d_out = (im.dt_area[d_sel] < a_rng[0]) | (im.dt_area[d_sel] > a_rng[1])
    dt_ig |= ~dtm & d_out[None, :]
    return {"dt_scores": im.dt_score[d_sel], "dt_matched": dtm, "dt_ignore": dt_ig, "gt_ignore": g_ig}


def evaluate(images, n_cat):
    """images: [ImageEval] -> {"precision": [T,R,K,A,M], "recall": [T,K,A,M], "stats": float[12]} (COCOeval.eval and .stats)."""
    images = sorted(images, key=lambda im: im.image_id)
    T, R, K, A, M = len(IOU_THRS), len(REC_THRS), int(n_cat), len(AREA_RNG), len(MAX_DETS)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    for k in range(K):
        for a, a_rng in enumerate(AREA_RNG):
            E = [e for e in (evaluate_img(im, k, a_rng) for im in images) if e is not None]
            if not E:
                continue
            gt_ig = np.concatenate([e["gt_ignore"] for e in E])
            npig = int(np.count_nonzero(~gt_ig))
            if npig == 0:
                continue
            for m, max_det in enumerate(MAX_DETS):
                scores = np.concatenate([e["dt_scores"][:max_det] for e in E])
                inds = np.argsort(-scores, kind="mergesort")
                dtm = np.concatenate([e["dt_matched"][:, :max_det] for e in E], axis=1)[:, inds]
                dt_ig = np.concatenate([e["dt_ignore"][:, :max_det] for e in E], axis=1)[:, inds]
                tp_sum = np.cumsum(dtm & ~dt_ig, axis=1).astype(np.float64)
                fp_sum = np.cumsum(~dtm & ~dt_ig, axis=1).astype(np.float64)
                for t in range(T):
                    tp, fp = tp_sum[t], fp_sum[t]
                    nd = len(tp)
                    rc = tp / npig
                    pr = tp / (fp + tp + np.spacing(1))
                    recall[t, k, a, m] = rc[-1] if nd else 0
                    pr = np.maximum.accumulate(pr[::-1])[::-1] if nd else pr
                    q = np.zeros(R)
                    idx = np.searchsorted(rc, REC_THRS, side="left")
                    ok = idx < nd
                    q[ok] = pr[idx[ok]]
                    precision[t, :, k, a, m] = q
    return {"precision": precision, "recall": recall, "stats": summarize(precision, recall)}


def _mean(s):
    s = s[s > -1]
    return float(np.mean(s)) if s.size else -1.0


def summarize(precision, recall):
    def ap(iou_thr=None, area="all", max_det=100):
        a, m = AREA_LBL.index(area), MAX_DETS.index(max_det)
        s = precision if iou_thr is None else precision[np.where(iou_thr == IOU_THRS)[0]]
        return _mean(s[:, :, :, a, m])

    def ar(area="all", max_det=100):
        return _mean(recall[:, :, AREA_LBL.index(area), MAX_DETS.index(max_det)])
    return np.array([ap(), ap(.5), ap(.75), ap(area="small"), ap(area="medium"), ap(area="large"), ar(max_det=1), ar(max_det=10), ar(),
                     ar("small"), ar("medium"), ar("large")])


def format_stats(stats):
    return "\n".join("%-6s %.4f" % (n, v) for n, v in zip(STAT_NAMES, stats))
