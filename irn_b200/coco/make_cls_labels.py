#!/usr/bin/env python
"""Build the MS COCO class-label dict the label-generation steps read (--coco_cls_labels) from an instances annotation file.

    python -m irn_b200.coco.make_cls_labels <coco_root>/annotations/instances_train2014.json coco/cls_labels.npy

Output: a .npy dict {stem: float32[80]}, in the format of voc12/cls_labels.npy.  The stem is the image's path relative to the COCO
root without its extension, ``<image_dir>/<file name>``, e.g. ``train2014/COCO_train2014_000000000009``; image_dir defaults to
what follows ``instances_`` in the annotation file's name.  Class k is the k-th category id of the file's ``categories`` in
ascending order (COCO's 80 ids lie between 1 and 90 with gaps).

- A crowd annotation (``iscrowd`` 1) counts like any other: its category is present in the image.
- An image without annotations gets an all-zero label; it stays in the dict, and make_cam writes it an empty CAM dict.

Only the ``json`` module reads the file (no pycocotools).
"""
import argparse
import json
import os

import numpy as np


def cls_labels(instances, image_dir):
    """instances: the parsed annotation file -> ({stem: float32[n_categories]}, sorted category ids)."""
    cat_ids = sorted(int(c["id"]) for c in instances["categories"])
    index = {c: k for k, c in enumerate(cat_ids)}
    stem = {}
    labels = {}
    for im in instances["images"]:
        s = image_dir + "/" + os.path.splitext(im["file_name"])[0]
        stem[int(im["id"])] = s
        labels[s] = np.zeros(len(cat_ids), np.float32)
    for a in instances["annotations"]:
        labels[stem[int(a["image_id"])]][index[int(a["category_id"])]] = 1.0
    return labels, cat_ids


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("instances_json")
    p.add_argument("out_npy")
    p.add_argument("--image_dir", default=None, help="directory of the images under the COCO root (default: from the file name)")
    a = p.parse_args(argv)
    image_dir = a.image_dir
    if image_dir is None:
        base = os.path.splitext(os.path.basename(a.instances_json))[0]
        image_dir = base[len("instances_"):] if base.startswith("instances_") else base
    with open(a.instances_json) as f:
        labels, cat_ids = cls_labels(json.load(f), image_dir)
    if os.path.dirname(a.out_npy):
        os.makedirs(os.path.dirname(a.out_npy), exist_ok=True)
    np.save(a.out_npy, labels)
    print("%d images, %d categories -> %s" % (len(labels), len(cat_ids), a.out_npy))


if __name__ == "__main__":
    main()
