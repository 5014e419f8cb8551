#!/usr/bin/env python
"""Driver for the pseudo-label generation steps, flag-compatible with the reference's ``run_sample.py``.

Every flag name and default of the reference (run_sample.py:11-72) is accepted and the output directories are the same,
so the reference's evaluation steps (step/eval_cam.py, step/eval_sem_seg.py, step/eval_ins_seg.py) read
``result/cam/*.npy``, ``result/sem_seg/*.png`` and ``result/ins_seg/*.npy`` unchanged.  The four inference steps run here
(make_cam, cam_to_ir_label -- the CRF on the GPU, writing ``result/ir_label/*.png`` --, make_ins_seg_labels, make_sem_seg_labels),
in the reference's order; the evaluation passes run when VOC ground truth is present; the training passes are the reference's own.

Differences: --cam_network / --irn_network default to the irn_b200 modules; flags the reference declares without a type
(--beta, --exp_times, --*_bg_thres, --*_pass) are parsed; --synthetic N runs on N seeded synthetic images instead of VOC
(--synthetic_list names them); --step_batch N images are processed together (of
any sizes in make_sem_seg_labels / make_ins_seg_labels / cam_to_ir_label, of one size in make_cam except for buckets
flushed before they fill, which take smaller images along; 1 = the reference's loop); --device_jpeg True decodes the JPEG
files the exact device decoder supports on the GPU, bit-identical to the host decode, so every output file is the same.

MS COCO: --dataset coco reads the images named in the lists (path stems relative to --coco_root, one per line) and their class
labels from --coco_cls_labels (irn_b200/coco/make_cls_labels.py builds it); the class count comes from the CAM checkpoint (80);
--irn_crop_size 640 takes COCO's largest images; eval_cam and eval_sem_seg score --infer_list against the class-index PNGs in
--coco_gt_dir over 81 classes, and eval_ins_seg scores the instance labels by COCO mask AP against --coco_instances (an
instances_*.json; the pass runs only when that file exists).

Threshold sweeps: --sweep_cam_pass True (after eval_cam) scores the CAMs at every background level of --cam_eval_thres_sweep,
--sweep_sem_seg_pass True (after eval_sem_seg) the semantic labels at every --sem_seg_bg_thres_sweep (one IRNet forward and one walk
per evaluation image for all of them); each prints one mIoU line per threshold and the best one.  Both flags take a comma list or
lo:hi:step (default 0.05:0.95:0.01); both passes are off by default and, like the evaluators, run only where ground truth is present.

--make_cocoann_pass True (default False: the reference's driver has no such pass) writes the instance labels of --infer_list as one
COCO annotation file, --cocoann_out (irn_b200/step/make_cocoann.py).
"""
import argparse
import os

from irn_b200.misc import pyutils
from irn_b200.step import _voc_eval


def _bool(v):
    return str(v).lower() in ("1", "true", "yes", "y")


def _device_jpeg(v):
    """--device_jpeg False (host decode) / True (the exact device decoder); `exact` is accepted as a spelling of True."""
    return str(v).lower() == "exact" or _bool(v)


def _dataset(v):
    v = str(v).lower()
    if v not in ("voc12", "coco"):
        raise argparse.ArgumentTypeError("--dataset is voc12 or coco, got %r" % v)
    return v


def _scales(v):
    return tuple(float(t) for t in str(v).split(","))


def _thresholds(v):
    """A threshold sweep's candidates: a comma list, or lo:hi:step (irn_b200.step._voc_eval.parse_thresholds)."""
    try:
        return tuple(_voc_eval.parse_thresholds(str(v)))
    except ValueError as e:
        raise argparse.ArgumentTypeError(str(e))


# (flag, default, type) in the reference's order: environment, dataset, CAM, relation mining, IRNet, random walk, outputs
FLAGS = [
    ("num_workers", os.cpu_count() // 2, int), ("dataset", "voc12", _dataset), ("voc12_root", "", str), ("coco_root", "", str),
    ("coco_cls_labels", "coco/cls_labels.npy", str), ("coco_gt_dir", "", str), ("coco_instances", "", str), ("synthetic", 0, int), ("synthetic_list", "", str), ("device_pyramid", True, _bool), ("device_jpeg", False, _device_jpeg),
    ("step_batch", 32, int),
    ("train_list", "voc12/train_aug.txt", str), ("val_list", "voc12/val.txt", str), ("infer_list", "voc12/train.txt", str),
    ("chainer_eval_set", "train", str),
    ("cam_network", "irn_b200.cam", str), ("cam_crop_size", 512, int), ("cam_batch_size", 16, int), ("cam_num_epoches", 5, int),
    ("cam_learning_rate", 0.1, float), ("cam_weight_decay", 1e-4, float), ("cam_eval_thres", 0.15, float),
    ("cam_eval_thres_sweep", _voc_eval.DEFAULT_SWEEP, _thresholds),
    ("cam_scales", (1.0, 0.5, 1.5, 2.0), _scales),
    ("conf_fg_thres", 0.30, float), ("conf_bg_thres", 0.05, float),
    ("irn_network", "irn_b200.irn", str), ("irn_crop_size", 512, int), ("irn_batch_size", 32, int), ("irn_num_epoches", 3, int),
    ("irn_learning_rate", 0.1, float), ("irn_weight_decay", 1e-4, float),
    ("beta", 10, float), ("exp_times", 8, int), ("ins_seg_bg_thres", 0.25, float), ("sem_seg_bg_thres", 0.25, float),
    ("sem_seg_bg_thres_sweep", _voc_eval.DEFAULT_SWEEP, _thresholds),
    ("log_name", "sample_train_eval", str), ("cam_weights_name", "sess/res50_cam.pth", str),
    ("irn_weights_name", "sess/res50_irn.pth", str), ("cam_out_dir", "result/cam", str), ("ir_label_out_dir", "result/ir_label", str),
    ("sem_seg_out_dir", "result/sem_seg", str), ("ins_seg_out_dir", "result/ins_seg", str),
    ("cocoann_out", "voc2012_train_custom.json", str),
]
PASSES = ["train_cam", "make_cam", "eval_cam", "sweep_cam", "cam_to_ir_label", "train_irn", "make_ins_seg", "eval_ins_seg", "make_sem_seg",
          "eval_sem_seg", "sweep_sem_seg", "make_cocoann"]
PASS_DEFAULT_OFF = {"sweep_cam", "sweep_sem_seg", "make_cocoann"}     # not passes of the reference's driver
HOT_STEPS = {"make_cam": "make_cam", "cam_to_ir_label": "cam_to_ir_label", "make_ins_seg": "make_ins_seg_labels",
             "make_sem_seg": "make_sem_seg_labels"}   # pass -> module
# evaluators and threshold sweeps: they run only where ground truth is present
EVAL_STEPS = {"eval_cam": "eval_cam", "eval_sem_seg": "eval_sem_seg", "eval_ins_seg": "eval_ins_seg", "sweep_cam": "sweep_cam",
              "sweep_sem_seg": "sweep_sem_seg"}


def parse(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    for name, default, typ in FLAGS:
        p.add_argument("--" + name, default=default, type=typ)
    for name in PASSES:
        p.add_argument("--%s_pass" % name, default=name not in PASS_DEFAULT_OFF, type=_bool)
    return p.parse_args(argv)


def _has_ground_truth(args, eval_pass):
    if args.dataset == "coco":       # class-index PNGs in --coco_gt_dir; instances in --coco_instances
        if eval_pass == "eval_ins_seg":
            return os.path.isfile(args.coco_instances)
        return os.path.isdir(args.coco_gt_dir)
    return os.path.isdir(os.path.join(args.voc12_root, "SegmentationClass"))


def main(argv=None):
    args = parse(argv)
    for d in ("sess", args.cam_out_dir, args.ir_label_out_dir, args.sem_seg_out_dir, args.ins_seg_out_dir):
        os.makedirs(d, exist_ok=True)
    pyutils.Logger(args.log_name + ".log")
    print(vars(args))
    if args.synthetic:   # no VOC data / trained checkpoints: seeded synthetic checkpoints in the reference's format
        import torch
        from irn_b200 import synth
        for path, make in ((args.cam_weights_name + ".pth", synth.cam_state_dict), (args.irn_weights_name, synth.irn_state_dict)):
            if not os.path.exists(path):
                torch.save(make(), path)
    import importlib
    for name in PASSES:
        if not getattr(args, name + "_pass"):
            continue
        if name in EVAL_STEPS and not args.synthetic and _has_ground_truth(args, name):
            pyutils.Timer("step.%s:" % name)
            importlib.import_module("irn_b200.step." + EVAL_STEPS[name]).run(args)
            continue
        if name == "make_cocoann":
            importlib.import_module("irn_b200.step.make_cocoann").run(args)
            continue
        if name not in HOT_STEPS:
            print("[irn_b200] step.%s is outside the native hot path: run the reference's own step for it" % name)
            continue
        module = importlib.import_module("irn_b200.step." + HOT_STEPS[name])
        pyutils.Timer("step.%s:" % HOT_STEPS[name])
        module.run(args)


if __name__ == "__main__":
    main()
