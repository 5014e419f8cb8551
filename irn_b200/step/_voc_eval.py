"""Ground-truth access and the confusion-matrix IoU the reference's evaluation steps use, without chainercv
(N2 in SURVEY.md section 8(f)).

chainercv's VOCSemanticSegmentationDataset reads `ImageSets/Segmentation/<split>.txt` and the palette PNGs under
`SegmentationClass/` (index 255 = ignore -> -1); calc_semantic_segmentation_confusion counts (gt, pred) pairs over the
pixels with gt >= 0.  Both are restated here in numpy.
"""
import os

import numpy as np
from PIL import Image


def voc_seg_ids(voc12_root, split):
    with open(os.path.join(voc12_root, "ImageSets", "Segmentation", split + ".txt")) as f:
        return [l.strip() for l in f if l.strip()]


def voc_seg_label(voc12_root, img_id):
    lab = np.asarray(Image.open(os.path.join(voc12_root, "SegmentationClass", img_id + ".png"))).astype(np.int32)
    lab[lab == 255] = -1
    return lab


def eval_set(args):
    """(image ids, ground-truth class-index maps with -1 = ignore, n_class) of the evaluation set: VOC's --chainer_eval_set split
    (21 classes), or with --dataset coco the images of --infer_list, whose ground truth is <--coco_gt_dir>/<name>.png (class index,
    255 = ignore) over 81 classes."""
    if str(getattr(args, "dataset", "voc12") or "voc12") != "coco":
        ids = voc_seg_ids(args.voc12_root, args.chainer_eval_set)
        return ids, [voc_seg_label(args.voc12_root, i) for i in ids], 21
    from ..coco import dataloader as coco_data
    ids = [os.path.basename(s) for s in coco_data.load_stem_list(args.infer_list)]
    labels = []
    for i in ids:
        lab = np.asarray(Image.open(os.path.join(args.coco_gt_dir, i + ".png"))).astype(np.int32)
        lab[lab == 255] = -1
        labels.append(lab)
    return ids, labels, coco_data.N_CAT + 1


def confusion(preds, labels, n_class=21):
    """rows = ground truth, cols = prediction; pixels with label < 0 are ignored (step/eval_sem_seg.py:18)."""
    conf = np.zeros((n_class, n_class), np.int64)
    for p, l in zip(preds, labels):
        p = np.asarray(p).reshape(-1).astype(np.int64)
        l = np.asarray(l).reshape(-1).astype(np.int64)
        ok = l >= 0
        if (p[ok] >= n_class).any() or (l[ok] >= n_class).any():
            raise ValueError("label outside [0, %d)" % n_class)
        conf += np.bincount(n_class * l[ok] + p[ok], minlength=n_class * n_class).reshape(n_class, n_class)
    return conf


def iou_from_confusion(conf):
    """step/eval_sem_seg.py:20-26: per-class IoU plus the false-positive / false-negative rates it prints."""
    gtj, resj, diag = conf.sum(axis=1), conf.sum(axis=0), np.diag(conf)
    with np.errstate(divide="ignore", invalid="ignore"):
        denom = gtj + resj - diag
        return {"iou": diag / denom, "fp": 1.0 - gtj / denom, "fn": 1.0 - resj / denom}


# ----------------------------------------------------------------------------- instance segmentation (step/eval_ins_seg.py)
def voc_instances(voc12_root, img_id):
    """chainercv VOCInstanceSegmentationDataset: SegmentationObject ids (0 = background and 255 = boundary are dropped) ->
    bool masks [R,H,W]; class of an instance = SegmentationClass value under its mask, minus 1 (0-based, 20 classes)."""
    cls = np.asarray(Image.open(os.path.join(voc12_root, "SegmentationClass", img_id + ".png"))).astype(np.int32)
    obj = np.asarray(Image.open(os.path.join(voc12_root, "SegmentationObject", img_id + ".png"))).astype(np.int32)
    cls[cls == 255] = -1
    obj[(obj == 0) | (obj == 255)] = -1
    masks, labels = [], []
    for i in np.unique(obj):
        if i == -1:
            continue
        m = obj == i
        masks.append(m)
        labels.append(int(np.unique(cls[m])[0]) - 1)
    if not masks:
        return np.zeros((0,) + obj.shape, bool), np.zeros((0,), np.int32)
    return np.stack(masks), np.asarray(labels, np.int32)


def mask_iou(a, b):
    """bool [N,H,W] x [K,H,W] -> float [N,K]."""
    a2 = a.reshape(len(a), -1).astype(np.float64)
    b2 = b.reshape(len(b), -1).astype(np.float64)
    inter = a2 @ b2.T
    union = a2.sum(1)[:, None] + b2.sum(1)[None] - inter
    with np.errstate(divide="ignore", invalid="ignore"):
        return inter / union


def instance_ap(pred_masks, pred_labels, pred_scores, gt_masks, gt_labels, iou_thresh=0.5):
    """chainercv.evaluations.eval_instance_segmentation_voc (use_07_metric=False), restated: per class, detections of
    each image in descending score take the ground-truth mask of highest IoU if that IoU >= iou_thresh and the mask is
    still free; AP = area under the monotone precision envelope.  Returns {"ap": float[n_class] (nan where a class has
    no ground truth), "map": nanmean}."""
    n_pos, score, match = {}, {}, {}
    for pm, pl, ps, gm, gl in zip(pred_masks, pred_labels, pred_scores, gt_masks, gt_labels):
        pl, ps, gl = np.asarray(pl), np.asarray(ps), np.asarray(gl)
        for l in np.unique(np.concatenate([pl, gl]).astype(int)):
            sel = pl == l
            order = np.argsort(-ps[sel], kind="stable")
            pm_l, ps_l = np.asarray(pm)[sel][order], ps[sel][order]
            gm_l = np.asarray(gm)[gl == l]
            n_pos[l] = n_pos.get(l, 0) + len(gm_l)
            score.setdefault(l, []).extend(ps_l.tolist())
            match.setdefault(l, [])
            if len(pm_l) == 0:
                continue
            if len(gm_l) == 0:
                match[l].extend([0] * len(pm_l))
                continue
            iou = mask_iou(pm_l, gm_l)
            gt_index = iou.argmax(axis=1)
            gt_index[iou.max(axis=1) < iou_thresh] = -1
            taken = np.zeros(len(gm_l), bool)
            for g in gt_index:
                if g >= 0 and not taken[g]:
                    match[l].append(1)
                    taken[g] = True
                else:
                    match[l].append(0)
                    if g >= 0:
                        taken[g] = True
    n_class = max(n_pos) + 1 if n_pos else 0
    ap = np.full(n_class, np.nan)
    for l in range(n_class):
        if n_pos.get(l, 0) == 0:
            continue
        order = np.argsort(-np.asarray(score[l]), kind="stable")
        m = np.asarray(match[l], np.int64)[order]
        tp, fp = np.cumsum(m == 1), np.cumsum(m == 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            prec = tp / (fp + tp)
        rec = tp / n_pos[l]
        mpre = np.concatenate([[0.0], np.nan_to_num(prec), [0.0]])
        mrec = np.concatenate([[0.0], rec, [1.0]])
        mpre = np.maximum.accumulate(mpre[::-1])[::-1]
        i = np.where(mrec[1:] != mrec[:-1])[0]
        ap[l] = np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])
    return {"ap": ap, "map": float(np.nanmean(ap)) if n_class else float("nan")}
