"""Drop-in for the reference's ``step/eval_cam.py``: mIoU of the thresholded high-resolution CAMs in
``result/cam/*.npy`` against VOC ground truth, without chainercv (step/eval_cam.py:7-29)."""
import os

import numpy as np

from . import _voc_eval


def run(args):
    ids, labels, n_class = _voc_eval.eval_set(args)
    preds = []
    for i in ids:
        d = np.load(os.path.join(args.cam_out_dir, i + ".npy"), allow_pickle=True).item()
        cams = np.pad(d["high_res"], ((1, 0), (0, 0), (0, 0)), mode="constant", constant_values=args.cam_eval_thres)
        keys = np.pad(np.asarray(d["keys"]) + 1, (1, 0), mode="constant")
        preds.append(keys[np.argmax(cams, axis=0)])
    r = _voc_eval.iou_from_confusion(_voc_eval.confusion(preds, labels, n_class))
    out = {"iou": r["iou"], "miou": np.nanmean(r["iou"])}
    print(out)
    return out
