"""The slice of the reference's ``voc12/dataloader.py`` the label-generation steps use (C1): image-name lists,
class labels, TorchvisionNormalize and the multi-scale + flip dataset, plus a synthetic stand-in for boxes
without VOC data."""
import os

import numpy as np
import torch
from PIL import Image
from torch.utils.data import Dataset

from ..misc import imutils

IMG_FOLDER_NAME = "JPEGImages"
N_CAT = 20

_cls_labels = {}


def cls_labels_dict(path="voc12/cls_labels.npy"):
    """voc12/dataloader.py:24 loads this dict at import time from the cwd; here it is loaded on first use."""
    if path not in _cls_labels:
        _cls_labels[path] = np.load(path, allow_pickle=True).item()
    return _cls_labels[path]


def decode_int_filename(int_filename):
    """voc12/dataloader.py:26-28 (also accepts the already-decoded 'YYYY_NNNNNN' form)."""
    s = str(int(str(int_filename).replace("_", "")))
    return s[:4] + "_" + s[4:]


def load_img_name_list(dataset_path):
    """voc12/dataloader.py:58-62 -- ids like 2007_000032 read as the integer 2007000032 (numpy>=2 safe)."""
    with open(dataset_path) as f:
        return np.array([int(l.strip().replace("_", "")) for l in f if l.strip()], dtype=np.int64)


def get_img_path(img_name, voc12_root):
    if not isinstance(img_name, str):
        img_name = decode_int_filename(img_name)
    return os.path.join(voc12_root, IMG_FOLDER_NAME, img_name + ".jpg")


class TorchvisionNormalize:
    """voc12/dataloader.py:65-78."""

    def __init__(self, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
        self.mean, self.std = mean, std

    def __call__(self, img):
        a = np.asarray(img)
        out = np.empty_like(a, np.float32)
        for c in range(3):
            out[..., c] = (a[..., c] / 255. - self.mean[c]) / self.std[c]
        return out


def multi_scale_flip(img_u8, scales, normalize=TorchvisionNormalize()):
    """voc12/dataloader.py:191-201: per scale -> PIL bicubic rescale, normalise, CHW, stack with the W-flip.
    Returns a list of float32 [2,3,h_s,w_s] (a single array when len(scales) == 1)."""
    out = []
    for s in scales:
        im = img_u8 if s == 1 else imutils.pil_rescale(img_u8, s, order=3)
        chw = imutils.HWC_to_CHW(normalize(im))
        out.append(np.stack([chw, np.flip(chw, -1)], axis=0))
    return out[0] if len(scales) == 1 else out


class VOC12ClassificationDatasetMSF(Dataset):
    """voc12/dataloader.py:175-205.  Items: {"name": str, "img": list of [2,3,h,w] (or one array),
    "size": (H, W), "label": FloatTensor[20]}."""

    def __init__(self, img_name_list_path, voc12_root, img_normal=TorchvisionNormalize(), scales=(1.0,),
                 cls_labels_path="voc12/cls_labels.npy", decode_only=False, raw_jpeg=False, cam_dir=None, cam_field="cam"):
        self.cam_field = cam_field          # which map of the CAM dict the worker ships (attach_cam)
        self.decode_only = decode_only      # hand over the decoded uint8 image; the pyramid is built on the device
        self.raw_jpeg = raw_jpeg            # hand over the FILE BYTES; nvJPEG decodes them on the device (irn_b200.jpeg)
        self.cam_dir = cam_dir              # label steps: the loader worker also reads the image's stored CAM dict (make_cam's .npy)
        self.img_name_list = load_img_name_list(img_name_list_path)
        self.voc12_root = voc12_root
        self.img_normal = img_normal
        self.scales = scales
        labels = cls_labels_dict(cls_labels_path)
        self.label_list = np.array([labels[int(n)] for n in self.img_name_list])

    def __len__(self):
        return len(self.img_name_list)

    def __getitem__(self, idx):
        name_str = decode_int_filename(self.img_name_list[idx])
        if self.raw_jpeg:
            path = get_img_path(name_str, self.voc12_root)
            with Image.open(path) as im:        # header only: the size decides the batch bucket
                w, h = im.size
                is_jpeg = im.format == "JPEG" and im.mode == "RGB"
            if is_jpeg:
                with open(path, "rb") as f:
                    data = np.frombuffer(f.read(), dtype=np.uint8).copy()
                return attach_cam({"name": name_str, "size": (h, w), "label": torch.from_numpy(self.label_list[idx]), "jpeg": data}, self.cam_dir, self.cam_field)
            # not a 3-component JPEG (grey-scale / PNG stand-ins): decode on the host like the reference
        img = np.asarray(Image.open(get_img_path(name_str, self.voc12_root)).convert("RGB"))
        out = {"name": name_str, "size": (img.shape[0], img.shape[1]), "label": torch.from_numpy(self.label_list[idx])}
        if self.decode_only:
            out["img_u8"] = np.array(img)            # writable copy: torch's collate wraps it without a warning
        else:
            out["img"] = multi_scale_flip(img, self.scales, self.img_normal)
        attach_cam(out, self.cam_dir, self.cam_field)
        return out


def attach_cam(item, cam_dir, field="cam"):
    """The label steps read `np.load(cam_out_dir/<name>.npy).item()` per image in their main loop
    (step/make_sem_seg_labels.py:34-37); with `cam_dir` set the loader WORKER does that read, in parallel with the decode, and
    ships what the steps use of it: `cam_keys` int64 [K] and, as item["cam"], the dict's `field`: the strided `cam` fp32
    [K,h/4,w/4] for the random-walk steps, the full-resolution `high_res` fp32 [K,H,W] for cam_to_ir_label."""
    if cam_dir:
        d = np.load(os.path.join(cam_dir, item["name"] + ".npy"), allow_pickle=True).item()
        item["cam_keys"] = torch.as_tensor(np.asarray(d["keys"]), dtype=torch.int64)
        item["cam"] = torch.as_tensor(np.asarray(d[field]), dtype=torch.float32).contiguous()
    return item


class SyntheticMSF(Dataset):
    """Same item format as VOC12ClassificationDatasetMSF over seeded synthetic images (irn_b200.synth):
    ids are taken from an image-name list when given, else 2007_000000 + index."""

    def __init__(self, n_items, size=(512, 512), scales=(1.0,), name_list=None, img_normal=TorchvisionNormalize(), decode_only=False,
                 cam_dir=None, cam_field="cam"):
        self.cam_dir, self.cam_field = cam_dir, cam_field
        self.decode_only = decode_only       # (no module stored on the instance: shards are pickled for spawn / DataLoader workers)
        self.n, self.size, self.scales, self.img_normal = n_items, size, scales, img_normal
        self.names = None if name_list is None else load_img_name_list(name_list)[:n_items]

    def __len__(self):
        return self.n

    def __getitem__(self, idx):
        name = decode_int_filename(self.names[idx]) if self.names is not None else "2007_%06d" % idx
        from .. import synth
        img = synth.image(idx, *self.size)
        out = {"name": name, "size": tuple(self.size), "label": torch.from_numpy(synth.label(idx))}
        if self.decode_only:
            out["img_u8"] = np.array(img)
        else:
            out["img"] = multi_scale_flip(img, self.scales, self.img_normal)
        return attach_cam(out, self.cam_dir, self.cam_field)
