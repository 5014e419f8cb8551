"""eval_cam at every threshold of --cam_eval_thres_sweep in one pass: each stored CAM is read once, and the confusion matrices of all
thresholds are counted on the device (indexing.ThresholdSweep).  Row j of the result is what eval_cam returns with
--cam_eval_thres thresholds[j]."""
import os

import numpy as np
import torch

from .. import indexing
from . import _common, _voc_eval


def missing_cams(ids, cam_out_dir):
    """Raise FileNotFoundError naming the evaluation images without a stored CAM."""
    missing = [i for i in ids if not os.path.isfile(os.path.join(cam_out_dir, i + ".npy"))]
    if missing:
        raise FileNotFoundError("no stored CAM in %s for evaluation image(s) %s" % (cam_out_dir, ", ".join(missing[:10])))


def upload_gt(device, gts):
    """uint8 ground-truth maps -> device tensors, staged through pinned memory."""
    return [torch.from_numpy(np.array(g, dtype=np.uint8)).pin_memory().to(device, non_blocking=True) for g in gts]


def run(args):
    thresholds = _voc_eval.parse_thresholds(getattr(args, "cam_eval_thres_sweep", _voc_eval.DEFAULT_SWEEP))
    ids, n_class = _voc_eval.eval_ids(args)
    missing_cams(ids, args.cam_out_dir)
    if not torch.cuda.is_available():
        raise RuntimeError("sweep_cam needs a CUDA device (there is no CPU fallback)")
    device = torch.device("cuda", torch.cuda.current_device())
    sweep = indexing.ThresholdSweep(thresholds, n_class, device)
    ctx = _common.StepContext(None, args, device, (1.0,))
    bsz = _common.step_batch(args)
    try:
        with torch.cuda.device(device):
            for o in range(0, len(ids), bsz):
                names = ids[o:o + bsz]
                stored = ctx.writer.map(lambda i: np.load(os.path.join(args.cam_out_dir, i + ".npy"), allow_pickle=True).item(), names)
                gts = upload_gt(device, ctx.writer.map(lambda i: _voc_eval.gt_png(args, i), names))
                cams = _common.to_device_list(ctx, [np.asarray(s["high_res"], np.float32) for s in stored])
                for cam, s, g in zip(cams, stored, gts):
                    sweep.add_cam(cam, np.asarray(s["keys"]), g)
            conf = sweep.confusion()
    finally:
        ctx.writer.close()
        ctx._copy_pool.shutdown()
    return _voc_eval.sweep_scores(sweep.thresholds, conf)
