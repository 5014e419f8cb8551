"""Drop-in for the reference's ``step/eval_sem_seg.py`` (mIoU of ``result/sem_seg/*.png`` against VOC ground truth)
without chainercv: same inputs, same printed quantities (step/eval_sem_seg.py:8-31)."""
import os

import numpy as np
from PIL import Image

from . import _voc_eval


def run(args):
    ids, labels, n_class = _voc_eval.eval_set(args)
    preds = []
    for i in ids:
        p = np.asarray(Image.open(os.path.join(args.sem_seg_out_dir, i + ".png"))).astype(np.uint8).copy()
        p[p == 255] = 0                                                   # step/eval_sem_seg.py:15
        preds.append(p)
    conf = _voc_eval.confusion(preds, labels, n_class)
    r = _voc_eval.iou_from_confusion(conf)
    print(r["fp"][0], r["fn"][0])
    print(np.mean(r["fp"][1:]), np.mean(r["fn"][1:]))
    out = {"iou": r["iou"], "miou": np.nanmean(r["iou"])}
    print(out)
    return out
