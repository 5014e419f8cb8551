"""The reference's ``step/make_cocoann.py``: the instance pseudo-labels ``result/ins_seg/*.npy`` of --infer_list as one COCO
annotation file (--cocoann_out, default ``voc2012_train_custom.json``), for training an instance segmentation network such as Mask
R-CNN on them.

Layout as the reference's: ``images`` (id, file_name, width, height and pycococreatortools' other image fields), ``annotations``,
``categories``, ``type: "instances"``; detections with score < 1e-5 are skipped; ``area`` and ``bbox`` are pycocotools' ``area`` and
``toBbox`` of the mask (irn_b200/coco/mask.py restates both); a mask without pixels is skipped (pycococreatortools'
create_annotation_info returns None for it, which the reference then writes as null).  Image ids: PASCAL VOC ``int(name[:4] +
name[5:])``, as the reference; MS COCO (--dataset coco) the id of the image in --coco_instances.

It deviates from the reference in four places:
  - segmentation is uncompressed RLE ({"counts", "size"}, column-major, the first run of zeros) with ``iscrowd`` 0.  The reference
    writes polygons, which need skimage's contour tracer and pycococreatortools, neither of them pinned here.  RLE is lossless and
    pycocotools-based loaders read it; Detectron2 needs ``INPUT.MASK_FORMAT bitmask``;
  - ``category_id`` is the dataset's category id (VOC class k -> k+1, COCO class k -> the k-th category id in ascending order).  The
    reference writes the 0-based class index against 1-based VOC categories;
  - annotation ids are unique over the file (1, 2, ... in image order).  The reference restarts them at 1 per image, and pycocotools'
    index then keeps only the last annotation of each id;
  - the categories are built in: VOC's 20 names with ids 1..20 instead of the reference's unshipped ``pascal_val2012.json``; COCO's
    are --coco_instances' own.
Host numpy only: the step is paced by the .npy reads."""
import json
import os

import numpy as np
from PIL import Image

from ..coco import mask as coco_mask
from . import _common

VOC_CATEGORIES = ("aeroplane", "bicycle", "bird", "boat", "bottle", "bus", "car", "cat", "chair", "cow", "diningtable", "dog", "horse",
                  "motorbike", "person", "pottedplant", "sheep", "sofa", "train", "tvmonitor")
DEFAULT_OUT = "voc2012_train_custom.json"
MIN_SCORE = 1e-5


def _images(args):
    """[(item name, image id, file name, H, W)] of --infer_list, and the categories, and class index -> category id."""
    if _common.dataset_name(args) == "coco":
        from ..coco.dataloader import load_stem_list
        from ..coco.make_cls_labels import category_index
        with open(args.coco_instances) as f:
            inst = json.load(f)
        cat_ids, _ = category_index(inst)
        by_name = {os.path.splitext(im["file_name"])[0]: im for im in inst["images"]}
        out = []
        for s in load_stem_list(args.infer_list):
            n = os.path.basename(s)
            if n not in by_name:
                raise KeyError("image %s of the list is not in %s" % (n, args.coco_instances))
            im = by_name[n]
            out.append((n, int(im["id"]), im["file_name"], int(im["height"]), int(im["width"])))
        cats = sorted(inst["categories"], key=lambda c: int(c["id"]))
        return out, cats, cat_ids
    from ..voc12 import dataloader as voc_data
    out = []
    for i in voc_data.load_img_name_list(args.infer_list):
        n = voc_data.decode_int_filename(i)
        with Image.open(voc_data.get_img_path(n, args.voc12_root)) as im:
            W, H = im.size
        out.append((n, int(n[:4] + n[5:]), n + ".jpg", H, W))
    return out, [{"supercategory": "none", "id": k + 1, "name": c} for k, c in enumerate(VOC_CATEGORIES)], list(range(1, 21))


def annotation_file(images, categories, cat_ids, ins_seg_out_dir):
    """The COCO dict of the detections stored for `images` ([(name, id, file name, H, W)])."""
    coco = {"images": [], "annotations": [], "categories": categories, "type": "instances"}
    ann_id = 1
    for name, img_id, file_name, H, W in images:
        coco["images"].append({"id": img_id, "file_name": file_name, "width": W, "height": H, "date_captured": "", "license": 1,
                               "coco_url": "", "flickr_url": ""})
        det = np.load(os.path.join(ins_seg_out_dir, name + ".npy"), allow_pickle=True).item()
        masks = np.asarray(det["mask"])
        if masks.shape[1:] != (H, W):
            raise ValueError("image %s: masks of shape %s, the image is %dx%d" % (name, masks.shape, H, W))
        for score, m, cls in zip(det["score"], masks, det["class"]):
            if score < MIN_SCORE:
                continue
            rle = coco_mask.rle_encode(m)
            area = coco_mask.rle_area(rle)
            if area < 1:
                continue
            coco["annotations"].append({"id": ann_id, "image_id": img_id, "category_id": int(cat_ids[int(cls)]), "iscrowd": 0,
                                        "area": area, "bbox": coco_mask.rle_bbox(rle), "segmentation": rle, "width": W, "height": H})
            ann_id += 1
    return coco


def run(args):
    images, categories, cat_ids = _images(args)
    coco = annotation_file(images, categories, cat_ids, args.ins_seg_out_dir)
    out = getattr(args, "cocoann_out", None) or DEFAULT_OUT
    if os.path.dirname(out):
        os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        json.dump(coco, f)
    print("%d images, %d annotations -> %s" % (len(coco["images"]), len(coco["annotations"]), out))
    return coco
