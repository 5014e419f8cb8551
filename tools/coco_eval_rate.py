#!/usr/bin/env python
"""Rate of the MS COCO instance evaluation (step/eval_ins_seg.py --dataset coco) on a synthetic COCO-shaped set.

    python tools/coco_eval_rate.py [--images 256] [--preds 30] [--gts 7] [--step_batch 32]

Writes, under a temporary directory, an instances JSON (polygon ground truth, every fifth annotation an uncompressed RLE crowd region)
and one ``.npy`` of bool masks [M,H,W] per image at COCO sizes, then runs the evaluation and prints images/s with the time split
between the JSON load, the .npy loads, the device (CUDA events around rasterisation, packing and overlaps), the host matching and
accumulation, and the card with its power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = [(480, 640), (640, 480), (427, 640), (640, 427), (375, 500), (612, 612), (640, 640), (333, 500)]


def _polygon(rng, h, w):
    cx, cy, r = rng.uniform(0, w), rng.uniform(0, h), rng.uniform(8, min(h, w) / 3)
    k = rng.randint(6, 40)
    a = np.sort(rng.uniform(0, 2 * np.pi, k))
    rr = r * rng.uniform(0.5, 1.0, k)
    return np.stack([cx + rr * np.cos(a), cy + rr * np.sin(a)], 1).reshape(-1).round(2).tolist()


def make_set(root, n, n_pred, n_gt, seed=0):
    from irn_b200.coco import mask as cmask
    rng = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, "ins_seg"), exist_ok=True)
    images, anns, stems = [], [], []
    yy_cache = {}
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        name = "COCO_val2014_%012d" % (i + 1)
        images.append({"id": i + 1, "file_name": name + ".jpg", "height": h, "width": w})
        stems.append("val2014/" + name)
        for j in range(n_gt):
            if j % 5 == 4:
                m = np.zeros((h, w), bool)
                y0, x0 = rng.randint(0, h // 2), rng.randint(0, w // 2)
                m[y0:y0 + h // 3, x0:x0 + w // 3] = True
                seg, crowd = cmask.rle_encode(m), 1
                area = float(m.sum())
            else:
                seg, crowd = [_polygon(rng, h, w)], 0
                area = float(rng.uniform(100, h * w / 4))
            anns.append({"id": len(anns) + 1, "image_id": i + 1, "category_id": 1 + rng.randint(80), "segmentation": seg, "area": area,
                         "iscrowd": crowd, "bbox": [0, 0, 0, 0]})
        if (h, w) not in yy_cache:
            yy_cache[(h, w)] = np.mgrid[0:h, 0:w]
        yy, xx = yy_cache[(h, w)]
        masks = np.zeros((n_pred, h, w), bool)
        for m in range(n_pred):
            cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(4, min(h, w) / 4)
            masks[m] = (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
        np.save(os.path.join(root, "ins_seg", name + ".npy"), {"score": rng.rand(n_pred).astype(np.float32), "mask": masks,
                                                                "class": rng.randint(0, 80, n_pred)})
    inst = {"images": images, "annotations": anns, "categories": [{"id": c, "name": str(c)} for c in range(1, 81)]}
    with open(os.path.join(root, "instances.json"), "w") as f:
        json.dump(inst, f)
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(stems) + "\n")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("--images", type=int, default=256)
    p.add_argument("--preds", type=int, default=30)
    p.add_argument("--gts", type=int, default=7)
    p.add_argument("--step_batch", type=int, default=32)
    a = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("coco_eval_rate needs a CUDA device")
    from irn_b200.coco import cocoeval
    from irn_b200.coco.dataloader import load_stem_list
    from irn_b200.step import eval_ins_seg
    with tempfile.TemporaryDirectory() as root:
        make_set(root, a.images, a.preds, a.gts)
        args = types.SimpleNamespace(dataset="coco", infer_list=os.path.join(root, "list.txt"), ins_seg_out_dir=os.path.join(root, "ins_seg"),
                                     coco_instances=os.path.join(root, "instances.json"), step_batch=a.step_batch)
        dev = torch.device("cuda", 0)
        names = [os.path.basename(s) for s in load_stem_list(args.infer_list)]
        # warm-up: one batch (module load, first launches)
        with open(args.coco_instances) as f:
            n_cat, gt = eval_ins_seg.coco_ground_truth(json.load(f), names)
        eval_ins_seg.coco_image_evals(args, gt[:a.step_batch], names[:a.step_batch], dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with open(args.coco_instances) as f:
            n_cat, gt = eval_ins_seg.coco_ground_truth(json.load(f), names)
        t_json = time.perf_counter() - t0
        timing = {}
        evals = eval_ins_seg.coco_image_evals(args, gt, names, dev, timing)
        t1 = time.perf_counter()
        stats = cocoeval.evaluate(evals, n_cat)["stats"]
        t_acc = time.perf_counter() - t1
        total = time.perf_counter() - t0
    name, pl = card()
    print("card: %s, power limit %s" % (name, pl))
    print("%d images (%d predictions, %d ground truths each), --step_batch %d: %.1f images/s (%.2f s)" %
          (a.images, a.preds, a.gts, a.step_batch, a.images / total, total))
    print("  json load %.3f s, npy load %.3f s, device %.3f s, host inputs %.3f s, matching + accumulation %.3f s, other %.3f s" %
          (t_json, timing["npy"], timing["device"], timing["host"], t_acc,
           total - t_json - timing["npy"] - timing["device"] - timing["host"] - t_acc))
    print("  AP %.4f (synthetic set: the value only shows the run finished)" % stats[0])


if __name__ == "__main__":
    main()
