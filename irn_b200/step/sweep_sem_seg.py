"""make_sem_seg_labels + eval_sem_seg at every threshold of --sem_seg_bg_thres_sweep in one pass: one IRNet forward and one random walk
per evaluation image (make_sem_seg_labels' own front half, walk_batch), then the confusion matrices of all background thresholds
counted on the device from the walk (indexing.ThresholdSweep) instead of one label map.  Row j of the result is what eval_sem_seg
returns after make_sem_seg_labels with --sem_seg_bg_thres thresholds[j].

With several GPUs each rank sums its stride shard; the ranks' confusion matrices, exact integers, are added up here."""
import functools
import glob
import os
import tempfile

import numpy as np
import torch

from .. import indexing
from . import _common, _voc_eval, make_sem_seg_labels, sweep_cam


def eval_list_path(args):
    """The image list of the evaluation set (_voc_eval.eval_ids): VOC's ImageSets/Segmentation/<--chainer_eval_set>.txt, or
    --infer_list with --dataset coco."""
    if _common.dataset_name(args) == "coco":
        return args.infer_list
    return os.path.join(args.voc12_root, "ImageSets", "Segmentation", args.chainer_eval_set + ".txt")


def _work(out_dir, thresholds, n_class, process_id, model, dataset, args):
    device = torch.device("cuda", process_id)
    sweep = indexing.ThresholdSweep(thresholds, n_class, device)

    def per_image(model, pack, args):
        name, keys, walk = make_sem_seg_labels.walk_one_image(model, pack, args)
        (gt,) = sweep_cam.upload_gt(device, [_voc_eval.gt_png(args, name)])
        sweep.add_walk(walk, keys, pack["size"], gt)

    def per_batch(ctx, packs):
        names, keys, rws, sizes = make_sem_seg_labels.walk_batch(ctx, packs)
        gts = sweep_cam.upload_gt(device, ctx.writer.map(lambda n: _voc_eval.gt_png(args, n), names))
        for rw, k, size, gt in zip(rws, keys, sizes, gts):
            sweep.add_walk(rw, k, size, gt)

    _common.work_loop(process_id, model, dataset, args, per_image, per_batch, ragged=True)
    with torch.cuda.device(device):
        np.save(os.path.join(out_dir, "rank%d.npy" % process_id), sweep.confusion())


def run(args):
    ids, n_class = _voc_eval.eval_ids(args)
    sweep_cam.missing_cams(ids, args.cam_out_dir)
    thresholds = indexing.ThresholdSweep(_voc_eval.parse_thresholds(getattr(args, "sem_seg_bg_thres_sweep", _voc_eval.DEFAULT_SWEEP)), n_class,
                                         "cuda").thresholds
    with tempfile.TemporaryDirectory() as out_dir:
        _common.run_step(args, functools.partial(_work, out_dir, thresholds, n_class), args.irn_network, "EdgeDisplacement",
                         args.irn_weights_name, False, eval_list_path(args), (1.0,), opening="[", cam_dir=args.cam_out_dir,
                         model_kwargs={"crop_size": int(getattr(args, "irn_crop_size", 512))})
        parts = sorted(glob.glob(os.path.join(out_dir, "rank*.npy")))
        if len(parts) != max(torch.cuda.device_count(), 1):
            raise RuntimeError("sweep_sem_seg: %d of %d ranks returned their counts" % (len(parts), torch.cuda.device_count()))
        conf = sum(np.load(p) for p in parts)
    return _voc_eval.sweep_scores(thresholds, conf, sem_seg=True)
