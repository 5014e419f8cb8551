"""COCO instance evaluation on the GPU: ground-truth rasterisation and prediction packing against oracle/coco_mask.py bit for bit, overlap
and area counts against numpy exactly, and eval_ins_seg / make_cocoann on a synthetic COCO tree."""
import json
import os
import types

import numpy as np
import pytest
import torch
from PIL import Image

from irn_b200 import synth
from irn_b200.coco import cocoeval
from irn_b200.coco import mask as cmask
from oracle import coco_mask as ocm

pytestmark = pytest.mark.gpu


def _random_polygon(rng, h, w, kind):
    if kind == "thin":          # a long thin sliver across the image
        x0, y0 = rng.uniform(-2, w + 2), rng.uniform(-2, h + 2)
        x1, y1 = rng.uniform(-2, w + 2), rng.uniform(-2, h + 2)
        d = rng.uniform(0.1, 1.5)
        return [x0, y0, x1, y1, x1 + d, y1 + d, x0 + d, y0]
    k = rng.randint(3, 12)
    if kind == "half":          # integral and half-integral vertices
        pts = rng.randint(-2, 2 * max(h, w) + 2, size=2 * k) / 2.0
    elif kind == "outside":     # vertices well off the image, some slightly negative
        pts = rng.uniform(-0.3 * max(h, w), 1.3 * max(h, w), size=2 * k)
        pts[rng.rand(2 * k) < 0.2] = -rng.uniform(0, 0.3)
    else:                       # arbitrary order: self-intersecting in general
        pts = np.stack([rng.uniform(0, w, k), rng.uniform(0, h, k)], 1).reshape(-1)
    return pts.tolist()


def _segmentations(rng, h, w, n):
    out = []
    for i in range(n):
        r = i % 5
        if r == 4:      # crowd-style uncompressed RLE
            m = rng.rand(h, w) < rng.uniform(0.05, 0.9)
            out.append(cmask.rle_encode(m))
        else:
            polys = [_random_polygon(rng, h, w, ("thin", "half", "outside", "free")[(i + j) % 4]) for j in range(1 + (i % 3 == 2))]
            out.append(polys)
    return out


def _device_masks(planes, offs, sizes):
    """Unpack device planes to bool masks through the oracle's layout."""
    host = planes.cpu().numpy().view(np.uint32)
    return [host[offs[i]:offs[i + 1]] for i in range(len(sizes))]


SIZES = [(1, 1), (1, 37), (29, 1), (375, 500), (640, 640), (33, 64), (500, 375)]


def test_rasterise_equals_oracle_and_ragged_equals_one_image(cuda_dev):
    rng = np.random.RandomState(3)
    anns = []
    for h, w in SIZES:
        for s in _segmentations(rng, h, w, 10):
            anns.append((h, w, s, len(anns)))
    planes, offs = cmask.rasterize(anns, cuda_dev)
    got = _device_masks(planes, offs, anns)
    for i, (h, w, s, _) in enumerate(anns):
        want = ocm.pack(ocm.ann_mask(s, h, w))
        assert np.array_equal(got[i], want), (i, h, w)
    nonempty = sum(int(ocm.ann_mask(s, h, w).any()) for h, w, s, _ in anns)
    assert nonempty > len(anns) // 2
    for i in rng.choice(len(anns), 12, replace=False):        # one annotation at a time gives the same bits
        p1, o1 = cmask.rasterize([anns[i]], cuda_dev)
        assert np.array_equal(p1.cpu().numpy().view(np.uint32), got[i])


def test_rasterise_edge_cases(cuda_dev):
    anns = [(10, 12, [[2, 3, 6, 3, 6, 8, 2, 8]], 1), (10, 12, [[1, 1, 5, 5]], 2), (10, 12, [[]], 3), (10, 12, [], 4),
            (10, 12, [[-3, -0.2, 20, -0.2, 20, 4, -3, 4], [1, 1, 1, 1, 6, 6]], 5), (64, 3, [[0, 0, 3, 0, 3, 64, 0, 64]], 6),
            (7, 5, {"counts": [0, 35], "size": [7, 5]}, 7), (7, 5, {"counts": [35], "size": [7, 5]}, 8)]
    planes, offs = cmask.rasterize(anns, cuda_dev)
    got = _device_masks(planes, offs, anns)
    for i, (h, w, s, _) in enumerate(anns):
        assert np.array_equal(got[i], ocm.pack(ocm.ann_mask(s, h, w))), i
    with pytest.raises(ValueError, match="annotation 99"):
        cmask.rasterize([(4, 4, {"counts": "abc", "size": [4, 4]}, 99)], cuda_dev)
    empty, o = cmask.rasterize([], cuda_dev)
    assert empty.numel() == 0


def _upload(masks, dev):
    return torch.from_numpy(np.concatenate([m.reshape(-1).view(np.uint8) for m in masks] + [np.zeros(0, np.uint8)])).to(dev)


def test_pack_and_overlaps_equal_numpy_counts(cuda_dev):
    rng = np.random.RandomState(5)
    cases = [(375, 500, 12, 7), (640, 640, 300, 3), (1, 1, 2, 1), (1, 37, 0, 4), (29, 1, 5, 0), (333, 500, 0, 0), (480, 640, 40, 9),
             (64, 32, 3, 17)]
    preds, gts = [], []
    for h, w, M, G in cases:
        preds.append(rng.rand(M, h, w) < rng.uniform(0.01, 0.6))
        gts.append(rng.rand(G, h, w) < rng.uniform(0.01, 0.6))
    pp = cmask.pack_masks(_upload(preds, cuda_dev), [(h, w, M) for h, w, M, G in cases])
    gp = cmask.pack_masks(_upload(gts, cuda_dev), [(h, w, G) for h, w, M, G in cases])
    want_pp = np.concatenate([ocm.pack(m) for p in preds for m in p])
    assert np.array_equal(pp.cpu().numpy().view(np.uint32), want_pp)
    out = cmask.overlaps(pp, gp, cases)
    for (inter, ap, ag), p, g in zip(out, preds, gts):
        wi, wa, wg = ocm.overlaps(p, g)
        assert inter.shape == wi.shape and np.array_equal(inter, wi) and np.array_equal(ap, wa) and np.array_equal(ag, wg)


# ------------------------------------------------------------------------------------------------ steps on a synthetic COCO tree
C = 80
TREE_SIZES = [(640, 480), (480, 640), (427, 640), (375, 500), (333, 500), (480, 640)]


@pytest.fixture(scope="module")
def coco_eval_tree(tmp_path_factory, cuda_dev):
    from irn_b200.step import make_cam, make_ins_seg_labels
    root = tmp_path_factory.mktemp("coco_eval")
    os.makedirs(root / "val2014")
    os.makedirs(root / "sess")
    stems, labels = [], {}
    for i, (h, w) in enumerate(TREE_SIZES):
        stem = "val2014/COCO_val2014_%012d" % (300 + i)
        Image.fromarray(synth.image(950 + i, h, w)).save(root / (stem + ".jpg"), quality=92)
        labels[stem] = synth.label(i, n_classes=C)
        stems.append(stem)
    np.save(root / "cls_labels.npy", labels)
    (root / "list.txt").write_text("\n".join(stems) + "\n")
    torch.save(synth.cam_state_dict(seed=5, n_classes=C), root / "sess" / "cam80.pth.pth")
    torch.save(synth.irn_state_dict(), root / "sess" / "irn.pth")
    args = _args(root, root / "out")
    make_cam.run(args)
    make_ins_seg_labels.run(args)
    # ground truth: polygons, uncompressed RLE and crowd regions of the images' own classes; category ids with gaps
    cat_ids = [1 + k + k // 7 for k in range(C)]
    rng = np.random.RandomState(11)
    images, anns = [], []
    for i, (stem, (h, w)) in enumerate(zip(stems, TREE_SIZES)):
        img_id = 1000 - 7 * i            # ids not in list order
        images.append({"id": img_id, "file_name": os.path.basename(stem) + ".jpg", "height": h, "width": w})
        det = np.load(os.path.join(args.ins_seg_out_dir, os.path.basename(stem) + ".npy"), allow_pickle=True).item()
        classes = np.flatnonzero(labels[stem])
        for j, s in enumerate(_segmentations(rng, h, w, 6)):
            crowd = isinstance(s, dict) and j % 2 == 1
            if j == 2 and len(det["mask"]):      # a ground truth equal to a detection, so some IoUs are 1
                s = cmask.rle_encode(np.asarray(det["mask"][0]))
                k = int(det["class"][0])
            else:
                k = int(classes[j % len(classes)])
            area = float(ocm.ann_mask(s, h, w).sum())
            anns.append({"id": len(anns) + 1, "image_id": img_id, "category_id": cat_ids[k], "segmentation": s, "area": area,
                         "iscrowd": int(crowd), "bbox": [0, 0, 0, 0]})
    inst = {"images": images, "annotations": anns, "categories": [{"id": c, "name": "c%d" % c} for c in cat_ids[::-1]]}
    (root / "instances_val2014.json").write_text(json.dumps(inst))
    return root, stems, args


def _args(root, out, **kw):
    a = dict(num_workers=0, dataset="coco", coco_root=str(root), coco_cls_labels=str(root / "cls_labels.npy"), coco_gt_dir="",
             coco_instances=str(root / "instances_val2014.json"), train_list=str(root / "list.txt"), infer_list=str(root / "list.txt"),
             cam_network="irn_b200.cam", irn_network="irn_b200.irn", cam_scales=(1.0, 0.5, 1.5, 2.0),
             cam_weights_name=str(root / "sess" / "cam80.pth"), irn_weights_name=str(root / "sess" / "irn.pth"), irn_crop_size=640,
             beta=10, exp_times=8, ins_seg_bg_thres=0.25, synthetic=0, step_batch=4, device_pyramid=True, device_jpeg=False,
             cocoann_out=str(out / "cocoann.json"))
    a.update(kw)
    for d in ("cam", "ir_label", "sem_seg", "ins_seg"):
        os.makedirs(out / d, exist_ok=True)
        a[d + "_out_dir"] = str(out / d)
    return types.SimpleNamespace(**a)


def _oracle_stats(inst, names, ins_dir):
    from irn_b200.coco.make_cls_labels import category_index
    cat_ids, index = category_index(inst)
    by_name = {os.path.splitext(im["file_name"])[0]: im for im in inst["images"]}
    evals = []
    for n in names:
        im = by_name[n]
        h, w = im["height"], im["width"]
        a = [x for x in inst["annotations"] if x["image_id"] == im["id"]]
        det = np.load(os.path.join(ins_dir, n + ".npy"), allow_pickle=True).item()
        gm = np.stack([ocm.ann_mask(x["segmentation"], h, w) for x in a]) if a else np.zeros((0, h, w), bool)
        inter, ap, ag = ocm.overlaps(np.asarray(det["mask"], bool), gm)
        evals.append(cocoeval.ImageEval(im["id"], [index[x["category_id"]] for x in a], [x["area"] for x in a],
                                        [bool(x["iscrowd"]) for x in a], ag, det["class"], det["score"], ap, inter))
    return cocoeval.evaluate(evals, len(cat_ids))


def test_eval_ins_seg_on_coco_equals_cocoeval_on_oracle_counts(coco_eval_tree):
    from irn_b200.step import eval_ins_seg
    root, stems, args = coco_eval_tree
    names = [os.path.basename(s) for s in stems]
    inst = json.loads((root / "instances_val2014.json").read_text())
    want = _oracle_stats(inst, names, args.ins_seg_out_dir)["stats"]
    assert (want > 0).any()
    for bsz in (4, 1, 32):
        got = eval_ins_seg.run(_args(root, root / "out", step_batch=bsz))
        assert np.array_equal(got, want), (bsz, got, want)


def test_make_cocoann_file_scores_its_own_labels_perfectly(coco_eval_tree, tmp_path):
    from irn_b200.step import eval_ins_seg, make_cocoann
    root, stems, args = coco_eval_tree
    a = _args(root, root / "out", cocoann_out=str(tmp_path / "ann.json"))
    coco = make_cocoann.run(a)
    assert coco["annotations"] and len({x["id"] for x in coco["annotations"]}) == len(coco["annotations"])
    inst = json.loads((root / "instances_val2014.json").read_text())
    assert {im["id"] for im in coco["images"]} == {im["id"] for im in inst["images"]}
    # the file as ground truth against the same .npy files: every detection it kept is its own match
    names = [os.path.basename(s) for s in stems]
    res = _oracle_stats(coco, names, args.ins_seg_out_dir)
    present = sorted({x["category_id"] for x in coco["annotations"]})
    from irn_b200.coco.make_cls_labels import category_index
    _, index = category_index(coco)
    ks = [index[c] for c in present]
    prec = res["precision"][:, :, ks, 0, 2]
    assert np.allclose(prec, 1.0, rtol=0, atol=1e-12), prec.min()
    assert np.allclose(res["recall"][:, ks, 0, 2], 1.0, rtol=0, atol=1e-12)
    a.coco_instances = a.cocoann_out
    got = eval_ins_seg.run(a)
    assert np.array_equal(got, res["stats"])
