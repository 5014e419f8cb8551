#!/usr/bin/env python
"""Rate of the semantic-label threshold sweep against make_sem_seg_labels on VOC-shaped input: a synthetic VOC tree (375 x 500 and
500 x 375 images, seeded ground truth, synthetic checkpoints) in a temporary directory, make_cam run once first.  Prints, in one run:
the card's name and power limit; images/s of make_sem_seg_labels, of sweep_sem_seg at T = 1 and at T = 91 (wall clock around
step.<name>.run, after a warm-up run of each, two rounds alternating); and the CUDA-event time per image of the sweep's accumulate
call against the walk's, on one 375 x 500 image with two classes.  Sets no target.

    python tools/sweep_rate.py --images 256 --step_batch 32
"""
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
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from irn_b200 import indexing, synth  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return "unknown"


def make_tree(root, n):
    for d in ("JPEGImages", "SegmentationClass", "ImageSets/Segmentation", "cam", "sem"):
        os.makedirs(os.path.join(root, d))
    ids, labels = [], {}
    for i in range(n):
        h, w = (375, 500) if i % 3 else (500, 375)
        name = "2007_%06d" % i
        Image.fromarray(synth.image(i, h, w)).save(os.path.join(root, "JPEGImages", name + ".jpg"), quality=90)
        labels[int(name.replace("_", ""))] = synth.label(i)
        gt = np.zeros((h, w), np.uint8)
        gt[h // 4:3 * h // 4, w // 4:3 * w // 4] = 1 + int(np.flatnonzero(synth.label(i))[0])
        Image.fromarray(gt).save(os.path.join(root, "SegmentationClass", name + ".png"))
        ids.append(name)
    for f, sel in (("list.txt", ids), ("warm.txt", ids[:16])):
        with open(os.path.join(root, "ImageSets", "Segmentation", f), "w") as fh:
            fh.write("\n".join(sel) + "\n")
    torch.save(synth.cam_state_dict(), os.path.join(root, "cam.pth.pth"))
    torch.save(synth.irn_state_dict(), os.path.join(root, "irn.pth"))
    return ids, labels


def event_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--images", type=int, default=256)
    p.add_argument("--step_batch", type=int, default=32)
    p.add_argument("--num_workers", type=int, default=8)
    a = p.parse_args()
    from irn_b200.step import make_cam, make_sem_seg_labels, sweep_sem_seg
    from irn_b200.voc12 import dataloader
    with tempfile.TemporaryDirectory() as root:
        ids, labels = make_tree(root, a.images)
        dataloader._cls_labels["voc12/cls_labels.npy"] = labels
        seg = os.path.join(root, "ImageSets", "Segmentation")
        args = types.SimpleNamespace(
            num_workers=a.num_workers, voc12_root=root, train_list=os.path.join(seg, "list.txt"), infer_list=os.path.join(seg, "list.txt"),
            chainer_eval_set="list", cam_network="irn_b200.cam", irn_network="irn_b200.irn", cam_scales=(1.0, 0.5, 1.5, 2.0),
            cam_weights_name=os.path.join(root, "cam.pth"), irn_weights_name=os.path.join(root, "irn.pth"), cam_out_dir=os.path.join(root, "cam"),
            sem_seg_out_dir=os.path.join(root, "sem"), beta=10, exp_times=8, sem_seg_bg_thres=0.25, synthetic=0, step_batch=a.step_batch)
        make_cam.run(args)
        runs = {"make_sem_seg_labels": lambda x: make_sem_seg_labels.run(x),
                "sweep_sem_seg_T1": lambda x: sweep_sem_seg.run(types.SimpleNamespace(**vars(x), sem_seg_bg_thres_sweep=[0.25])),
                "sweep_sem_seg_T91": lambda x: sweep_sem_seg.run(types.SimpleNamespace(**vars(x), sem_seg_bg_thres_sweep="0.05:0.95:0.01"))}
        warm = types.SimpleNamespace(**vars(args))
        warm.chainer_eval_set, warm.infer_list = "warm", os.path.join(seg, "warm.txt")
        for fn in runs.values():
            fn(warm)
        rates = {k: [] for k in runs}
        for _ in range(2):
            for k, fn in runs.items():
                torch.cuda.synchronize()
                t = time.perf_counter()
                fn(args)
                torch.cuda.synchronize()
                rates[k].append(a.images / (time.perf_counter() - t))

    dev = torch.device("cuda:0")
    h, w, H, W = 94, 125, 375, 500
    x = torch.from_numpy(synth.seeds(2, h, w, 3)).to(dev)
    edge = torch.from_numpy(synth.edge_map(h, w, "bimodal", 3)).to(dev).reshape(1, h, w)
    gt = torch.randint(0, 21, (H, W), dtype=torch.uint8, device=dev)
    walk_ms = event_ms(lambda: indexing.random_walk_batch(x, edge, [0, 2], 5, 10.0, 256), 20)
    rw = indexing.random_walk_batch(x, edge, [0, 2], 5, 10.0, 256)
    out = {"card": card(), "images": a.images, "step_batch": a.step_batch,
           "images_per_s": {k: [round(v, 1) for v in r] for k, r in rates.items()},
           "walk_ms_per_image": round(walk_ms, 4)}
    for T in (1, 91):
        sweep = indexing.ThresholdSweep(np.linspace(0.05, 0.95, T) if T > 1 else [0.25], 21, dev)
        out["accumulate_ms_per_image_T%d" % T] = round(event_ms(lambda: sweep.add_walk(rw, [3, 9], (H, W), gt), 200), 4)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
