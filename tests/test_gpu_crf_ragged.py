"""Ragged CRF batches (irn_b200.crf.dense_crf_ragged / ir_labels_ragged, irn_dense_crf_ragged / irn_ir_label_ragged): images of any
sizes in one call give, bit for bit, what each image gives in its own one-size call; chunking, errors; cam_to_ir_label on mixed-size
VOC and COCO trees writes the same files with one ragged CRF call per batch as with the one-image loop."""
import ctypes
import hashlib
import os
import types

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import golden_path
from irn_b200 import _lib, crf, synth
from oracle import crf as ocrf

pytestmark = pytest.mark.gpu

G = np.load(golden_path("ir_label.npz"))
STEPS = np.load(golden_path("steps.npz"))


def _img(seed, h, w):
    return synth.image(seed, h, w) if h * w > 1 else np.array([[[(10 + seed) % 256, 20, 30]]], np.uint8)


def _flat(imgs, dev):
    return torch.from_numpy(np.concatenate([i.reshape(-1) for i in imgs])).to(dev), [i.shape[:2] for i in imgs]


# batches of (H, W) with one n_labels each: degenerate and odd sizes, VOC's two orientations, a COCO-sized 81-label image, 1 label
DENSE_BATCHES = {
    "odd": ([(1, 1), (1, 7), (9, 1), (3, 5), (13, 17), (20, 24), (1, 1)], 3),
    "voc": ([(375, 500), (500, 375), (37, 53)], 4),
    "coco81": ([(31, 47), (640, 640), (5, 3)], 81),
    "one_label": ([(7, 9), (16, 12), (1, 1)], 1),
}


@pytest.mark.parametrize("name", list(DENSE_BATCHES))
def test_dense_ragged_equals_per_image(cuda_dev, name):
    sizes, n = DENSE_BATCHES[name]
    imgs = [_img(40 + i, h, w) for i, (h, w) in enumerate(sizes)]
    labs = [np.random.RandomState(i).randint(0, n, (h, w)).astype(np.int32) for i, (h, w) in enumerate(sizes)]
    flat, sz = _flat(imgs, cuda_dev)
    lab_flat = torch.from_numpy(np.concatenate([l.reshape(-1) for l in labs])).to(cuda_dev)
    out, q, counts = crf.dense_crf_ragged(flat, sz, lab_flat, n, want_q=True)
    outs, qs = crf.unpack(out, sz), crf.unpack(q, sz, n)
    for i, (img, lab) in enumerate(zip(imgs, labs)):
        l1, q1, c1 = crf.dense_crf(torch.from_numpy(img)[None].to(cuda_dev), torch.from_numpy(lab)[None].to(cuda_dev), n, want_q=True)
        assert torch.equal(qs[i], q1[0]), (name, i)
        assert torch.equal(outs[i], l1[0]), (name, i)
        assert counts[i].tolist() == c1[0].tolist(), (name, i)
        if img.shape[0] * img.shape[1] <= 24 * 24:
            d = ocrf.DenseCRF2D(img.shape[1], img.shape[0], n)
            d.setUnaryEnergy(ocrf.unary_from_labels(lab, n, 0.7))
            d.addPairwiseGaussian(sxy=3, compat=3)
            d.addPairwiseBilateral(sxy=50, srgb=5, rgbim=img, compat=10)
            q_ref = d.inference(10).reshape(n, *img.shape[:2])
            assert counts[i].tolist() == [p.lattice.n_vertices for p in d.pairwise]
            assert float(np.abs(qs[i].cpu().numpy() - q_ref).max()) < 1e-5


def _golden(i):
    if ("seed%d" % i) in G:
        H, W = G["png%d" % i].shape
        u8 = synth.cam_planes_u8(len(G["keys%d" % i]), H, W, int(G["seed%d" % i]))
        assert hashlib.sha256(np.ascontiguousarray(u8).tobytes()).hexdigest() == str(G["cam_sha256%d" % i])
        return synth.image(int(G["seed%d" % i]), H, W), synth.u8_to_cam(u8), G["keys%d" % i]
    j = int(G["steps_index%d" % i])
    return STEPS["img%d" % j], STEPS["cam_high%d" % j].astype(np.float32), G["keys%d" % i]


def _synthetic(n_classes):
    """Seeded cases of mixed sizes and class counts (0 classes: one label) for a dataset of n_classes."""
    sizes = [(48, 64), (64, 48), (1, 1), (17, 5), (33, 40), (90, 70), (2, 9)]
    counts = [0, 1, 3, 2, 6, 1, 4]
    out = []
    for i, ((h, w), k) in enumerate(zip(sizes, counts)):
        keys = np.sort(np.random.RandomState(100 + i).choice(n_classes, k, replace=False))
        high = synth.u8_to_cam(synth.cam_planes_u8(k, h, w, 200 + i)) if k else np.zeros((0, h, w), np.float32)
        out.append((_img(300 + i, h, w), high, keys))
    return out


def _ragged_conf(cases, dev, n_classes=20, **kw):
    flat, sz = _flat([c[0] for c in cases], dev)
    out = crf.ir_labels_ragged(flat, sz, [c[1] for c in cases], [c[2] for c in cases], 0.30, 0.05, n_classes=n_classes, **kw)
    return [m.cpu().numpy() for m in crf.unpack(out, sz)]


def _alone(case, dev, n_classes=20):
    x = torch.from_numpy(case[0])[None].to(dev)
    return crf.ir_labels(x, [case[1]], [case[2]], 0.30, 0.05, n_classes=n_classes)[0].cpu().numpy()


@pytest.mark.parametrize("which", ["golden", "voc_synthetic", "coco_synthetic"])
def test_ir_labels_ragged_equals_per_image(cuda_dev, which):
    nc = 80 if which == "coco_synthetic" else 20
    cases = [_golden(i) for i in range(int(G["n"]))] if which == "golden" else _synthetic(nc)
    alone = [_alone(c, cuda_dev, nc) for c in cases]
    got = _ragged_conf(cases, cuda_dev, nc)
    for i in range(len(cases)):
        assert np.array_equal(got[i], alone[i]), (which, i)
    assert all(np.array_equal(a, b) for a, b in zip(_ragged_conf(cases, cuda_dev, nc), got))      # repeated calls: same bits
    # batch invariance: the same image first, last, and between other neighbours
    rev = _ragged_conf(cases[::-1], cuda_dev, nc)[::-1]
    mixed = _ragged_conf([cases[-1]] + cases + [cases[0]], cuda_dev, nc)[1:-1]
    for i in range(len(cases)):
        assert np.array_equal(rev[i], alone[i]) and np.array_equal(mixed[i], alone[i]), (which, i)


def test_ir_labels_ragged_chunks(cuda_dev):
    cases = _synthetic(20) + [_golden(0)]
    sz = [c[0].shape[:2] for c in cases]
    whole = _ragged_conf(cases, cuda_dev)
    per = [_lib.lib().irn_crf_ragged_workspace_bytes(1, np.array(s, np.int32).ctypes.data_as(ctypes.c_void_p), 2, 7) for s in sz]
    limit = 2 * max(per)
    assert len(crf._ragged_chunks(per, limit)) > 1
    chunked = _ragged_conf(cases, cuda_dev, max_workspace_bytes=limit)
    for a, b in zip(whole, chunked):
        assert np.array_equal(a, b)


def test_ragged_errors(cuda_dev):
    cases = _synthetic(20)[:3]
    flat, sz = _flat([c[0] for c in cases], cuda_dev)
    high, keys = [c[1] for c in cases], [c[2] for c in cases]
    with pytest.raises(_lib.IrnError, match="add up"):
        crf.ir_labels_ragged(torch.cat([flat, flat[:1]]), sz, high, keys, 0.3, 0.05)
    with pytest.raises(_lib.IrnError, match="add up"):
        crf.dense_crf_ragged(flat[:-3], sz, torch.zeros(sum(h * w for h, w in sz), dtype=torch.int32, device=cuda_dev), 2)
    bad = list(high)
    bad[1] = np.zeros((len(keys[1]),) + tuple(sz[1])[::-1], np.float32)
    with pytest.raises(_lib.IrnError, match="shape"):
        crf.ir_labels_ragged(flat, sz, bad, keys, 0.3, 0.05)
    with pytest.raises(_lib.IrnError, match="outside"):
        crf.ir_labels_ragged(flat, sz, high, [keys[0], np.array([20]), keys[2]], 0.3, 0.05)
    with pytest.raises(_lib.IrnError):
        crf.ir_labels_ragged(flat.cpu(), sz, high, keys, 0.3, 0.05)
    # the C entry points: wrong byte totals, bad sizes and a short workspace come back as return codes
    L = _lib.lib()
    hw = np.ascontiguousarray(np.array(sz, np.int32))
    nN = int(sum(h * w for h, w in sz))
    counts = np.array([len(k) for k in keys], np.int32)
    kk = np.ascontiguousarray(np.concatenate(keys).astype(np.int32))
    planes = torch.cat([torch.from_numpy(h).reshape(-1) for h in high]).to(cuda_dev)
    out = torch.empty(nN, dtype=torch.uint8, device=cuda_dev)
    need = L.irn_crf_ragged_workspace_bytes(3, hw.ctypes.data_as(ctypes.c_void_p), 2, int(counts.max()) + 1)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda_dev)

    def call(img_bytes=3 * nN, sizes=hw, elems=planes.numel(), ws_bytes=need):
        rc = L.irn_ir_label_ragged(_lib.ptr(flat), img_bytes, sizes.ctypes.data_as(ctypes.c_void_p), 3, _lib.ptr(planes), elems,
                                   kk.ctypes.data_as(ctypes.c_void_p), counts.ctypes.data_as(ctypes.c_void_p), 0.3, 0.05, _lib.ptr(out),
                                   None, _lib.ptr(ws), ws_bytes, _lib.stream_ptr())
        torch.cuda.synchronize()
        return rc
    assert call() == 0
    assert call(img_bytes=3 * nN - 3) == -1
    assert call(elems=planes.numel() + 1) == -1
    zero = hw.copy()
    zero[1, 0] = 0
    assert call(sizes=zero) == -1
    assert call(ws_bytes=need - 1) == -3
    assert L.irn_crf_ragged_workspace_bytes(3, zero.ctypes.data_as(ctypes.c_void_p), 2, 4) == 0


# ------------------------------------------------------------------------------------------------ the step on mixed-size trees
VOC_SIZES = [(375, 500), (500, 375), (333, 500), (500, 333), (375, 500), (281, 500), (97, 131), (500, 375), (120, 161), (500, 400)]
COCO_SIZES = [(480, 640), (640, 480), (427, 640), (640, 640), (360, 640), (640, 512), (480, 640), (612, 640), (398, 640)]


def _tree(root, dataset, sizes):
    """JPEG files, class labels, a list, and make_cam-style dicts (keys, high_res) for cam_to_ir_label."""
    nc = 80 if dataset == "coco" else 20
    rs = np.random.RandomState(len(sizes))
    names, stems, labels = [], [], {}
    os.makedirs(root / "cam")
    for i, (h, w) in enumerate(sizes):
        if dataset == "coco":
            stem = "train2014/COCO_train2014_%012d" % (500 + i)
            name = os.path.basename(stem)
        else:
            stem = name = "2008_%06d" % (10 + i)
            stem = "JPEGImages/" + stem
        os.makedirs(os.path.dirname(root / (stem + ".jpg")), exist_ok=True)
        Image.fromarray(synth.image(600 + i, h, w)).save(root / (stem + ".jpg"), quality=90)
        k = int(rs.randint(0, 7)) if dataset == "coco" else int(rs.randint(0, 4))
        keys = np.sort(rs.choice(nc, k, replace=False)).astype(np.int64)
        label = np.zeros(nc, np.float32)
        label[keys] = 1
        high = synth.u8_to_cam(synth.cam_planes_u8(k, h, w, 700 + i)) if k else np.zeros((0, h, w), np.float32)
        np.save(root / "cam" / (name + ".npy"), {"keys": keys, "high_res": high})
        names.append(name)
        stems.append(stem[len("JPEGImages/"):] if dataset != "coco" else stem)
        labels[stem if dataset == "coco" else int(name.replace("_", ""))] = label
    (root / "list.txt").write_text("\n".join(stems) + "\n")
    if dataset == "coco":
        np.save(root / "cls_labels.npy", labels)
    else:
        from irn_b200.voc12 import dataloader
        dataloader._cls_labels["voc12/cls_labels.npy"] = labels
    return names


def _run(root, dataset, out, **kw):
    from irn_b200.step import cam_to_ir_label
    a = dict(num_workers=0, dataset=dataset, train_list=str(root / "list.txt"), cam_out_dir=str(root / "cam"), conf_fg_thres=0.30,
             conf_bg_thres=0.05, synthetic=0, step_batch=32, device_pyramid=True, device_jpeg=False, ir_label_out_dir=str(out))
    if dataset == "coco":
        a.update(coco_root=str(root), coco_cls_labels=str(root / "cls_labels.npy"))
    else:
        a.update(voc12_root=str(root))
    a.update(kw)
    os.makedirs(out)
    cam_to_ir_label.run(types.SimpleNamespace(**a))


@pytest.mark.parametrize("dataset", ["voc12", "coco"])
def test_step_ragged_batches_write_the_one_image_files(cuda_dev, tmp_path, monkeypatch, dataset):
    sizes = COCO_SIZES if dataset == "coco" else VOC_SIZES
    assert len(set(sizes)) >= 6
    names = _tree(tmp_path, dataset, sizes)
    calls = []
    real = crf.ir_labels_ragged

    def spy(flat, sz, *a, **kw):
        calls.append([tuple(s) for s in sz])
        return real(flat, sz, *a, **kw)
    monkeypatch.setattr(crf, "ir_labels_ragged", spy)
    _run(tmp_path, dataset, tmp_path / "batched")
    monkeypatch.setattr(crf, "ir_labels_ragged", real)
    assert any(len(set(c)) > 1 for c in calls) and sum(len(c) for c in calls) == len(sizes)
    _run(tmp_path, dataset, tmp_path / "one", step_batch=1)
    _run(tmp_path, dataset, tmp_path / "dev", device_jpeg=True)
    for name, (h, w) in zip(names, sizes):
        ref = (tmp_path / "one" / (name + ".png")).read_bytes()
        assert (tmp_path / "batched" / (name + ".png")).read_bytes() == ref, name
        assert (tmp_path / "dev" / (name + ".png")).read_bytes() == ref, name
        assert np.asarray(Image.open(tmp_path / "one" / (name + ".png"))).shape == (h, w)
