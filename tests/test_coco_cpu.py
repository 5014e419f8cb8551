"""MS COCO on the host, no GPU: the class-label converter, the COCO loader's items, the --dataset flags, the packed parameter blob
of an 80-class CAM checkpoint, and the errors for a class count above 128, a class id the plan does not have and an image larger
than the IRNet crop."""
import ctypes
import json
import os
import types

import numpy as np
import pytest
import torch
from PIL import Image

from irn_b200 import _lib, _pack, synth
from irn_b200.cam import CAM, tap_shape
from irn_b200.coco import dataloader as coco_data
from irn_b200.coco import make_cls_labels
from irn_b200.irn import EdgeDisplacement
from irn_b200.step import _common, _voc_eval

# COCO's 80 category ids: 1..90 without 12, 26, 29, 30, 45, 66, 68, 69, 71, 83
CAT_IDS = [i for i in range(1, 91) if i not in (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)]


def _instances():
    cats = [{"id": c, "name": "c%d" % c} for c in reversed(CAT_IDS)]        # not sorted in the file
    images = [{"id": 9, "file_name": "COCO_train2014_000000000009.jpg", "height": 48, "width": 64},
              {"id": 25, "file_name": "COCO_train2014_000000000025.jpg", "height": 64, "width": 40},
              {"id": 30, "file_name": "COCO_train2014_000000000030.jpg", "height": 40, "width": 40}]
    anns = [{"id": 1, "image_id": 9, "category_id": 1, "iscrowd": 0},
            {"id": 2, "image_id": 9, "category_id": 90, "iscrowd": 0},
            {"id": 3, "image_id": 9, "category_id": 90, "iscrowd": 0},
            {"id": 4, "image_id": 25, "category_id": 13, "iscrowd": 1},        # crowd: counts
            {"id": 5, "image_id": 25, "category_id": 46, "iscrowd": 0}]
    return {"images": images, "annotations": anns, "categories": cats}            # image 30 has no annotation


@pytest.fixture(scope="module")
def coco_tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("coco")
    os.makedirs(root / "annotations")
    os.makedirs(root / "train2014")
    (root / "annotations" / "instances_train2014.json").write_text(json.dumps(_instances()))
    make_cls_labels.main([str(root / "annotations" / "instances_train2014.json"), str(root / "cls_labels.npy")])
    sizes = {9: (48, 64), 25: (64, 40), 30: (40, 40)}
    stems = []
    for i, (h, w) in sizes.items():
        stem = "train2014/COCO_train2014_%012d" % i
        img = synth.image(i, h, w)
        if i == 25:
            Image.fromarray(img[..., 0]).save(root / (stem + ".jpg"), quality=90)     # greyscale JPEG
        else:
            Image.fromarray(img).save(root / (stem + ".jpg"), quality=90)
        stems.append(stem)
    (root / "list.txt").write_text("\n".join(stems) + "\n")
    return root, stems, sizes


def test_converter_maps_ids_crowd_and_empty_images(coco_tree):
    root, stems, _ = coco_tree
    d = np.load(root / "cls_labels.npy", allow_pickle=True).item()
    assert sorted(d) == sorted(stems)
    for v in d.values():
        assert v.dtype == np.float32 and v.shape == (80,)
    assert np.flatnonzero(d[stems[0]]).tolist() == [0, 79]                       # ids 1 and 90: first and last class
    assert np.flatnonzero(d[stems[1]]).tolist() == [CAT_IDS.index(13), CAT_IDS.index(46)] == [11, 40]   # crowd annotation kept
    assert not d[stems[2]].any()                                                   # no annotation: all zero, still listed


def test_converter_image_dir_option(tmp_path):
    p = tmp_path / "a.json"
    p.write_text(json.dumps(_instances()))
    make_cls_labels.main([str(p), str(tmp_path / "o.npy"), "--image_dir", "val2014"])
    assert all(k.startswith("val2014/COCO_train2014_") for k in np.load(tmp_path / "o.npy", allow_pickle=True).item())


@pytest.mark.parametrize("decode_only", [True, False])
def test_loader_items(coco_tree, decode_only):
    root, stems, sizes = coco_tree
    ds = coco_data.COCOClassificationDatasetMSF(str(root / "list.txt"), coco_root=str(root), cls_labels_path=str(root / "cls_labels.npy"),
                                                scales=(1.0, 0.5), decode_only=decode_only)
    labels = np.load(root / "cls_labels.npy", allow_pickle=True).item()
    assert len(ds) == 3
    for k, stem in enumerate(stems):
        it = ds[k]
        i = int(stem[-12:])
        assert it["name"] == os.path.basename(stem) and it["size"] == sizes[i]
        assert it["label"].dtype == torch.float32 and it["label"].shape == (80,)
        assert np.array_equal(it["label"].numpy(), labels[stem])
        ref = np.asarray(Image.open(root / (stem + ".jpg")).convert("RGB"))
        if decode_only:
            assert np.array_equal(it["img_u8"], ref)                             # greyscale decoded to R = G = B
        else:
            assert [a.shape for a in it["img"]] == [(2, 3) + sizes[i], (2, 3, sizes[i][0] // 2, sizes[i][1] // 2)]


def test_loader_raw_bytes_match_decoded_pixels(coco_tree):
    """--device_jpeg: the worker ships the file bytes of every JPEG the exact decoder takes (greyscale included), with the size
    of the pixels the host decode gives."""
    root, stems, sizes = coco_tree
    ds = coco_data.COCOClassificationDatasetMSF(str(root / "list.txt"), coco_root=str(root), cls_labels_path=str(root / "cls_labels.npy"),
                                                decode_only=True, raw_jpeg=True)
    for k, stem in enumerate(stems):
        it = ds[k]
        assert "jpeg_exact" in it and "img_u8" not in it
        assert it["jpeg_exact"].tobytes() == (root / (stem + ".jpg")).read_bytes()
        assert it["size"] == np.asarray(Image.open(root / (stem + ".jpg")).convert("RGB")).shape[:2]


def test_loader_refuses_a_list_entry_without_label(coco_tree, tmp_path):
    root, stems, _ = coco_tree
    (tmp_path / "l.txt").write_text(stems[0] + "\ntrain2014/COCO_train2014_000000000777\n")
    with pytest.raises(KeyError, match="no class label"):
        coco_data.COCOClassificationDatasetMSF(str(tmp_path / "l.txt"), coco_root=str(root), cls_labels_path=str(root / "cls_labels.npy"))


def test_make_dataset_picks_coco(coco_tree):
    root, stems, _ = coco_tree
    args = types.SimpleNamespace(dataset="coco", coco_root=str(root), coco_cls_labels=str(root / "cls_labels.npy"), step_batch=4,
                                 device_pyramid=True, device_jpeg=False, synthetic=0)
    ds = _common.make_dataset(args, str(root / "list.txt"), (1.0,))
    assert isinstance(ds, coco_data.COCOClassificationDatasetMSF) and ds[0]["name"] == os.path.basename(stems[0])
    with pytest.raises(ValueError):
        _common.make_dataset(types.SimpleNamespace(**dict(vars(args), dataset="ade")), str(root / "list.txt"), (1.0,))


def test_coco_eval_set(coco_tree, tmp_path):
    root, stems, sizes = coco_tree
    for stem in stems:
        h, w = sizes[int(stem[-12:])]
        gt = np.full((h, w), 80, np.uint8)
        gt[0] = 255
        Image.fromarray(gt).save(tmp_path / (os.path.basename(stem) + ".png"))
    args = types.SimpleNamespace(dataset="coco", infer_list=str(root / "list.txt"), coco_gt_dir=str(tmp_path))
    ids, labels, n_class = _voc_eval.eval_set(args)
    assert ids == [os.path.basename(s) for s in stems] and n_class == 81
    assert all((l[0] == -1).all() and (l[1:] == 80).all() for l in labels)
    conf = _voc_eval.confusion([np.full(l.shape, 80) for l in labels], labels, n_class)
    assert conf.shape == (81, 81) and conf[80, 80] == sum(int((l >= 0).sum()) for l in labels)


def test_flags():
    import run_sample
    a = run_sample.parse([])
    assert (a.dataset, a.coco_root, a.coco_cls_labels, a.coco_gt_dir, a.irn_crop_size) == ("voc12", "", "coco/cls_labels.npy", "", 512)
    a = run_sample.parse(["--dataset", "coco", "--coco_root", "/data/coco", "--coco_gt_dir", "/data/gt", "--coco_cls_labels", "l.npy",
                          "--irn_crop_size", "640"])
    assert (a.dataset, a.coco_root, a.coco_gt_dir, a.coco_cls_labels, a.irn_crop_size) == ("coco", "/data/coco", "/data/gt", "l.npy", 640)
    with pytest.raises(SystemExit):
        run_sample.parse(["--dataset", "cityscapes"])


def test_voc_names_unchanged():
    from irn_b200.voc12 import dataloader as voc_data
    assert voc_data.decode_int_filename(2007000032) == voc_data.decode_int_filename("2007_000032") == "2007_000032"
    assert voc_data.decode_int_filename("COCO_val2014_000000000042") == "COCO_val2014_000000000042"


def test_cam_takes_class_count_from_checkpoint_and_packs_it():
    sd = synth.cam_state_dict(seed=3, n_classes=80)
    assert tuple(sd["classifier.weight"].shape) == (80, 2048, 1, 1)
    m = CAM()
    m.load_state_dict(sd, strict=True)
    assert m.n_classes == 80 and len(m.state_dict()) == 956
    blob = _pack.pack_cam(m.state_dict())
    trunk = _pack.pack_cam(synth.cam_state_dict(seed=3)).size - 20 * 2048
    assert blob.size == trunk + 80 * 2048
    assert np.array_equal(blob[trunk:], sd["classifier.weight"].numpy().reshape(-1))
    # and back to VOC: the synthetic 20-class checkpoint is what it always was
    m.load_state_dict(synth.cam_state_dict(), strict=True)
    assert m.n_classes == 20
    assert np.array_equal(synth.label(5, n_classes=20), synth.label(5))


def test_errors(built_lib):
    bad = synth.cam_state_dict(seed=3, n_classes=20)
    bad["classifier.weight"] = torch.zeros(129, 2048, 1, 1)
    with pytest.raises(_lib.IrnError, match="1..128"):
        CAM().load_state_dict(bad, strict=True)
    with pytest.raises(ValueError):
        CAM(0)
    L = _lib.lib()
    blob = np.zeros(16, np.float32)
    h = ctypes.c_void_p()
    assert L.irn_cam_net_create_classes(blob.ctypes.data, blob.size, 129, ctypes.byref(h)) != 0
    assert b"129 classes" in L.irn_last_error()
    assert L.irn_cam_workspace_bytes_classes(2, 64, 64, 129) == 0
    assert L.irn_cam_workspace_bytes_classes(2, 64, 64, 80) > L.irn_cam_workspace_bytes(2, 64, 64)
    # merge: a class id >= C, K > C and C > 128 are refused on the host, before the device pointers are touched
    ptrs = (ctypes.c_void_p * 1)(1)
    hs, ws = (ctypes.c_int * 1)(4), (ctypes.c_int * 1)(4)
    for n_classes, keys in ((80, [3, 80]), (20, [20]), (2, [0, 1, 1]), (129, [0])):
        k = np.asarray(keys, np.int32)
        assert L.irn_cam_merge_classes(ptrs, hs, ws, 1, n_classes, 64, 64, k.ctypes.data, k.size, ctypes.c_void_p(1), None,
                                       ctypes.c_void_p(1), None) == -1, (n_classes, keys)
    # an image larger than the IRNet crop is refused before any device work
    irn = EdgeDisplacement(crop_size=640)
    with pytest.raises(_lib.IrnError, match="larger than crop_size 640"):
        irn.forward_ragged(torch.zeros(641 * 480 * 3, dtype=torch.uint8), [(641, 480)])
    with pytest.raises(_lib.IrnError, match="larger than crop_size 512"):
        EdgeDisplacement().forward_ragged(torch.zeros(640 * 480 * 3, dtype=torch.uint8), [(480, 640)])


def test_tap_shape_follows_class_count(built_lib):
    assert tap_shape(0, 50, 4, 40, 72) == tap_shape(0, 50, 4, 40, 72, n_classes=64) == (4, 3, 5, 64)
    assert tap_shape(0, 50, 4, 40, 72, n_classes=80) == tap_shape(0, 50, 4, 40, 72, n_classes=128) == (4, 3, 5, 128)
    assert tap_shape(0, 0, 4, 40, 72, n_classes=80) == tap_shape(0, 0, 4, 40, 72)
    with pytest.raises(_lib.IrnError):
        tap_shape(0, 50, 4, 40, 72, n_classes=129)
