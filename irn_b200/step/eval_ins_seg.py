"""Drop-in for the reference's ``step/eval_ins_seg.py`` (AP at IoU 0.5 of ``result/ins_seg/*.npy`` against the VOC
instance ground truth) without chainercv: same inputs, same printed quantity (step/eval_ins_seg.py:7-23).  chainercv is
absent from this image, so the restated metric (irn_b200/step/_voc_eval.py::instance_ap) is checked on hand-computable
cases only: "parity unpinned" for this evaluator.

With --dataset coco the same files are scored by COCO mask AP (irn_b200/coco/cocoeval.py) against --coco_instances (an
``instances_*.json``, read with ``json`` only) over the images of --infer_list: an item is matched to the JSON image whose
``file_name`` without its extension is the stem's basename, and class k is the k-th category id in ascending order.  Every
--step_batch images, the ground truth is rasterised and every prediction/ground-truth overlap counted on the device
(irn_b200/coco/mask.py); matching and accumulation run on the host.  Prints and returns the 12 standard numbers."""
import json
import os
import time

import numpy as np
import torch

from . import _common, _voc_eval


def run(args):
    if _common.dataset_name(args) == "coco":
        return run_coco(args)
    ids = _voc_eval.voc_seg_ids(args.voc12_root, args.chainer_eval_set)
    gt = [_voc_eval.voc_instances(args.voc12_root, i) for i in ids]
    pred = [np.load(os.path.join(args.ins_seg_out_dir, i + ".npy"), allow_pickle=True).item() for i in ids]
    out = _voc_eval.instance_ap([p["mask"] for p in pred], [p["class"] for p in pred], [p["score"] for p in pred],
                                [g[0] for g in gt], [g[1] for g in gt], iou_thresh=0.5)
    print("0.5iou:", out)
    return out


def coco_ground_truth(instances, names):
    """The parsed annotation file and item names -> (number of classes, [(JSON image, its annotations, their class indices)] per name)."""
    from ..coco.make_cls_labels import category_index
    cat_ids, index = category_index(instances)
    by_name = {os.path.splitext(im["file_name"])[0]: im for im in instances["images"]}
    anns = {}
    for a in instances["annotations"]:
        anns.setdefault(int(a["image_id"]), []).append(a)
    out = []
    for n in names:
        if n not in by_name:
            raise KeyError("image %s of the list is not in the annotation file" % n)
        im = by_name[n]
        a = anns.get(int(im["id"]), [])
        out.append((im, a, np.array([index[int(x["category_id"])] for x in a], np.int64)))
    return len(cat_ids), out


class _Staging:
    """One pinned host buffer, grown to the largest batch, for the prediction masks' upload."""

    def __init__(self):
        self.buf = None

    def upload(self, arrays, device):
        n = sum(a.size for a in arrays)
        if self.buf is None or self.buf.numel() < n:
            self.buf = torch.empty(max(n, 1), dtype=torch.uint8).pin_memory()
        host = self.buf[:n].numpy()
        o = 0
        for a in arrays:
            host[o:o + a.size] = a.reshape(-1)
            o += a.size
        return self.buf[:n].to(device, non_blocking=True)


def coco_image_evals(args, gt, names, device, timing=None):
    """The cocoeval inputs of `names` (gt: coco_ground_truth's list), --step_batch images per device call.  timing: a dict that
    receives the seconds spent loading the .npy files ("npy"), on the device ("device", CUDA events) and building the inputs ("host")."""
    from ..coco import cocoeval, mask
    bsz = _common.step_batch(args)
    staging = _Staging()
    out = []
    t = timing if timing is not None else {}
    for k in ("npy", "device", "host"):
        t.setdefault(k, 0.0)
    for b0 in range(0, len(names), bsz):
        t0 = time.perf_counter()
        preds = [np.load(os.path.join(args.ins_seg_out_dir, n + ".npy"), allow_pickle=True).item() for n in names[b0:b0 + bsz]]
        t1 = time.perf_counter()
        t["npy"] += t1 - t0
        batch, masks, anns, hwmg = gt[b0:b0 + bsz], [], [], []
        for n, p, (im, a, _) in zip(names[b0:b0 + bsz], preds, batch):
            H, W = int(im["height"]), int(im["width"])
            m = np.asarray(p["mask"])
            if m.ndim != 3 or m.shape[1:] != (H, W):
                raise ValueError("image %s: prediction masks of shape %s, the annotation file says %dx%d" % (n, m.shape, H, W))
            masks.append(np.ascontiguousarray(m, bool).view(np.uint8))
            anns += [(H, W, x["segmentation"], x.get("id")) for x in a]
            hwmg.append((H, W, m.shape[0], len(a)))
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.device(device):
            ev0.record()
            gt_planes, _ = mask.rasterize(anns, device)
            pred_planes = mask.pack_masks(staging.upload(masks, device), [h[:3] for h in hwmg])
            counts = mask.overlaps(pred_planes, gt_planes, hwmg)
            ev1.record()
            ev1.synchronize()
        t["device"] += ev0.elapsed_time(ev1) / 1e3
        t2 = time.perf_counter()
        for p, (im, a, cls), (inter, area_p, area_g) in zip(preds, batch, counts):
            out.append(cocoeval.ImageEval(im["id"], cls, [float(x["area"]) for x in a], [bool(x.get("iscrowd", 0)) for x in a], area_g,
                                          np.asarray(p["class"]), np.asarray(p["score"]), area_p, inter))
        t["host"] += time.perf_counter() - t2
    return out


def run_coco(args):
    from ..coco import cocoeval
    from ..coco.dataloader import load_stem_list
    names = [os.path.basename(s) for s in load_stem_list(args.infer_list)]
    with open(args.coco_instances) as f:
        n_cat, gt = coco_ground_truth(json.load(f), names)
    device = torch.device("cuda", torch.cuda.current_device())
    stats = cocoeval.evaluate(coco_image_evals(args, gt, names, device), n_cat)["stats"]
    print(cocoeval.format_stats(stats))
    return stats
