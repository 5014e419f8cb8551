"""MS COCO for the label-generation steps: the same items as voc12.dataloader.VOC12ClassificationDatasetMSF (decode-only images,
raw JPEG bytes for the exact device decoder, the stored CAMs attached by the loader workers), over COCO's image list and class
labels.

  list file     one image per line as a path stem relative to --coco_root, e.g. ``train2014/COCO_train2014_000000000009``
  image         <coco_root>/<stem>.jpg
  item name     the stem's basename (``COCO_train2014_000000000009``): the steps name their output files after it
  class labels  a .npy dict {stem: float32[80]} (make_cls_labels.py builds it from annotations/instances_*.json), class k = the
                k-th COCO category id in ascending order
"""
import os

import numpy as np

from ..voc12 import dataloader as voc_data

N_CAT = 80


def load_stem_list(list_path):
    with open(list_path) as f:
        return [l.strip() for l in f if l.strip()]


class COCOClassificationDatasetMSF(voc_data.VOC12ClassificationDatasetMSF):
    """VOC12ClassificationDatasetMSF over MS COCO: only the list, the labels, the item names and the image paths differ."""

    def __init__(self, img_name_list_path, coco_root, cls_labels_path, **kw):
        super().__init__(img_name_list_path, voc12_root=coco_root, cls_labels_path=cls_labels_path, **kw)

    def _load_list(self, list_path, cls_labels_path):
        stems = load_stem_list(list_path)
        labels = voc_data.cls_labels_dict(cls_labels_path)
        missing = [s for s in stems if s not in labels]
        if missing:
            raise KeyError("%d images of %s have no class label in %s, e.g. %s" % (len(missing), list_path, cls_labels_path, missing[0]))
        return stems, np.array([np.asarray(labels[s], np.float32) for s in stems]).reshape(len(stems), -1)

    def item_name(self, idx):
        return os.path.basename(self.img_name_list[idx])

    def image_path(self, idx):
        return os.path.join(self.voc12_root, self.img_name_list[idx] + ".jpg")
