#!/usr/bin/env python
"""Rate of make_cam and make_sem_seg_labels on MS COCO-shaped input: a synthetic COCO tree (JPEG files in a temporary directory,
a list of path stems, an 80-class label dict) with COCO's size mix, 80-class checkpoints, --irn_crop_size 640.  Prints one JSON
line: images/s of each step (wall clock around step.<name>.run, after one warm-up run of each on the first 32 images), the card's
name and power limit, and which walk kernel a 160 x 160 feature grid runs on.  Sets no target.

    python tools/coco_rate.py --images 512 --step_batch 32
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

# long side 640 with the short side drawn from COCO's common heights/widths; a tenth square 640 x 640
SHORT_SIDES = (480, 427, 426, 424, 425, 428, 640, 360, 383, 512)


def coco_sizes(n, seed=0):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        s = int(SHORT_SIDES[rs.randint(len(SHORT_SIDES))])
        out.append((s, 640) if rs.rand() < 0.6 else (640, s))
    return out


def make_tree(root, sizes):
    os.makedirs(os.path.join(root, "train2014"))
    stems, labels = [], {}
    for i, (h, w) in enumerate(sizes):
        stem = "train2014/COCO_train2014_%012d" % i
        Image.fromarray(synth.image(i, h, w)).save(os.path.join(root, stem + ".jpg"), quality=90)
        labels[stem] = synth.label(i, n_classes=80)
        stems.append(stem)
    np.save(os.path.join(root, "cls_labels.npy"), labels)
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(stems) + "\n")
    with open(os.path.join(root, "warm.txt"), "w") as f:
        f.write("\n".join(stems[:32]) + "\n")
    torch.save(synth.cam_state_dict(seed=5, n_classes=80), os.path.join(root, "cam80.pth.pth"))
    torch.save(synth.irn_state_dict(), os.path.join(root, "irn.pth"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--step_batch", type=int, default=32)
    ap.add_argument("--num_workers", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("coco_rate needs a CUDA device")
    from irn_b200.step import make_cam, make_sem_seg_labels
    with tempfile.TemporaryDirectory() as root:
        make_tree(root, coco_sizes(a.images))
        out = {}
        for d in ("cam", "sem"):
            os.makedirs(os.path.join(root, d))
        args = types.SimpleNamespace(
            num_workers=a.num_workers, dataset="coco", coco_root=root, coco_cls_labels=os.path.join(root, "cls_labels.npy"),
            cam_network="irn_b200.cam", irn_network="irn_b200.irn", cam_scales=(1.0, 0.5, 1.5, 2.0),
            cam_weights_name=os.path.join(root, "cam80.pth"), irn_weights_name=os.path.join(root, "irn.pth"), irn_crop_size=640,
            cam_out_dir=os.path.join(root, "cam"), sem_seg_out_dir=os.path.join(root, "sem"), beta=10, exp_times=8,
            sem_seg_bg_thres=0.25, synthetic=0, step_batch=a.step_batch, device_pyramid=True, device_jpeg=False)
        for name, mod, lst in (("make_cam", make_cam, "train_list"), ("make_sem_seg_labels", make_sem_seg_labels, "infer_list")):
            setattr(args, "train_list", os.path.join(root, "warm.txt"))
            setattr(args, "infer_list", os.path.join(root, "warm.txt"))
            mod.run(args)
            setattr(args, lst, os.path.join(root, "list.txt"))
            torch.cuda.synchronize()
            t = time.perf_counter()
            mod.run(args)
            torch.cuda.synchronize()
            out[name + "_images_per_s"] = round(a.images / (time.perf_counter() - t), 2)
        e = torch.from_numpy(synth.edge_map(160, 160, "bimodal", 0)).cuda()
        indexing.random_walk_batch(torch.from_numpy(synth.seeds(2, 160, 160)).cuda(), e, [0, 2], 5, 10, 256)
        out["walk_kernel_160x160"] = "fused cluster" if indexing.last_walk_was_fused() else "per-step TMA"
        out.update(images=a.images, step_batch=a.step_batch, card=card())
        print(json.dumps(out))


if __name__ == "__main__":
    main()
