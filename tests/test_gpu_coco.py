"""MS COCO on the GPU: 80-class CAM networks, images up to 640 pixels, CRFs of up to 81 labels, and the four label steps on a
synthetic COCO tree.

  CAM (C = 80)   one-size and ragged forwards at the four make_cam scales, in conv modes 0, 1 and 2, against the float64 oracle on
                 the device within the 1e-4 max-normalised contract, on the synthetic and the trained-like checkpoints; ragged equals
                 one-size bit for bit; an integer-valued 2048 -> 128 classifier conv is exact in every mode
  merge          K = 1, 20, 21 and 80 keys of an 80-class CAM against oracle/steps.py
  IRNet          crop 640 against the float64 oracle (edge and dp within 1e-4); ragged equals one-size bit for bit
  walk           160 x 160 feature grids (beyond the fused cluster walk) within 2e-6 of the float64 oracle; the padded walk equals
                 the walk on the image's own grid bit for bit at exp_times 0 and 8
  CRF            22 to 81 labels against oracle/crf.py bit for bit; cam_to_ir_label for an image with 30 classes
  steps          make_cam -> cam_to_ir_label -> make_ins_seg_labels -> make_sem_seg_labels on a synthetic COCO tree: batched writes
                 what --step_batch 1 writes, --device_jpeg True what the host decode writes; eval_cam / eval_sem_seg match numpy
"""
import ctypes
import os
import types

import numpy as np
import pytest
import torch
from PIL import Image

import layer_check as lc
from irn_b200 import _lib, indexing, preprocess, synth
from irn_b200.cam import CAM
from irn_b200.irn import EdgeDisplacement
from irn_b200.pipeline import PseudoLabelPipeline
from oracle import crf as ocrf
from oracle import indexing as oi
from oracle import nets, steps

pytestmark = pytest.mark.gpu

C = 80
SIZES = [(640, 640), (480, 640), (640, 427), (375, 500)]
SCALES = (1.0, 0.5, 1.5, 2.0)


def _trained_like_cam(n_classes=C, seed=7):
    sd = lc.hostile_cam_state_dict(seed)
    g = torch.Generator().manual_seed(seed + 100)
    w = 0.01 * torch.randn((n_classes, 2048, 1, 1), generator=g)
    for k in ("classifier.weight", "newly_added.0.weight"):      # the checkpoint's two names of the classifier
        sd[k] = w.clone()
    return sd


CHECKPOINTS = {"synthetic": lambda: synth.cam_state_dict(seed=5, n_classes=C), "trained_like": _trained_like_cam}


def _sd64(sd, dev):
    return {k: v.to(dev, torch.float64) for k, v in sd.items() if v.dtype.is_floating_point}


@pytest.fixture(scope="module")
def images(cuda_dev):
    return [torch.from_numpy(synth.image(700 + i, h, w)).to(cuda_dev) for i, (h, w) in enumerate(SIZES)]


@pytest.mark.parametrize("ckpt", sorted(CHECKPOINTS))
def test_cam80_forward_vs_fp64_oracle_and_ragged_bitwise(cuda_dev, images, ckpt):
    sd = CHECKPOINTS[ckpt]()
    sd64 = _sd64(sd, cuda_dev)
    m = CAM()
    m.load_state_dict(sd, strict=True)
    assert m.n_classes == C
    worst = 0.0
    for s in SCALES:
        xs = [preprocess.resize_normalize(im, im.shape[:2] if s == 1 else preprocess.rescaled_size(*im.shape[:2], s)) for im in images]
        refs = [nets.cam_forward(x.double(), sd64) for x in xs]
        flat = torch.cat([im.reshape(-1) for im in images])
        canvas, ext = preprocess.resize_normalize_ragged(flat, SIZES, s)
        for mode in (0, 1, 2):
            m.set_conv_mode(mode)
            rag = m.forward_ragged(canvas, ext)
            assert rag.shape[:2] == (len(SIZES), C)
            for i, (x, ref) in enumerate(zip(xs, refs)):
                y = m(x)
                assert y.shape == ref.shape == (C, (x.shape[2] - 1) // 16 + 1, (x.shape[3] - 1) // 16 + 1)
                err = float((y.double() - ref).abs().max() / ref.max())
                worst = max(worst, err)
                assert err < 1e-4, "%s scale %g size %s mode %d: normalised err %g" % (ckpt, s, SIZES[i], mode, err)
                h, w = y.shape[1:]
                assert torch.equal(rag[i, :, :h, :w], y), (ckpt, s, SIZES[i], mode)
                assert not rag[i, :, h:].any() and not rag[i, :, :, w:].any()
    m.set_conv_mode(None)
    print("cam80 %s worst normalised err %.3g" % (ckpt, worst))


def test_cam80_classifier_conv_exact(cuda_dev):
    """The 80-class classifier as the tensor-core path runs it, a 2048 -> 128 1x1 conv with rows 80.. zero, on integer values whose
    products and sums are exact in every arithmetic: every mode returns the exact result."""
    rs = np.random.RandomState(0)
    w = np.zeros((128, 2048, 1, 1), np.float32)
    w[:C] = rs.randint(-2, 3, (C, 2048, 1, 1))
    x = rs.randint(-2, 3, (2, 5, 7, 2048)).astype(np.float32)
    ref = np.einsum("bhwc,oc->bhwo", x.astype(np.float64), w[:, :, 0, 0].astype(np.float64)).astype(np.float32)
    L = _lib.lib()
    h = ctypes.c_void_p()
    _lib.check(L.irn_conv_create(w.ctypes.data, None, 2048, 128, 1, 1, 0, ctypes.byref(h)), "irn_conv_create")
    try:
        xd = torch.from_numpy(x).to(cuda_dev)
        for mode in (0, 1, 2):
            out = torch.full((2, 5, 7, 128), float("nan"), device=cuda_dev)
            _lib.check(L.irn_conv_forward(h, _lib.ptr(xd), 2, 5, 7, None, _lib.ptr(out), 0, mode, _lib.stream_ptr()), "irn_conv_forward")
            assert np.array_equal(out.cpu().numpy(), ref), mode
    finally:
        L.irn_conv_destroy(h)


@pytest.mark.parametrize("K", [1, 20, 21, 80])
def test_merge_k_of_80(cuda_dev, K):
    from irn_b200 import cam_ops
    rs = np.random.RandomState(K)
    H, W = 427, 640
    outs = [torch.from_numpy(rs.rand(C, hs, ws).astype(np.float32)) for hs, ws in ((27, 40), (14, 20), (41, 60), (54, 80))]
    label = np.zeros(C, np.float32)
    label[rs.choice(C, K, replace=False)] = 1
    keys, lo, hi = cam_ops.merge_cams([o.to(cuda_dev) for o in outs], (H, W), torch.from_numpy(label))
    rk, rlo, rhi = steps.cam_merge(outs, (H, W), torch.from_numpy(label))
    assert np.array_equal(keys.numpy(), rk.numpy()) and keys.numel() == K
    assert (lo.cpu() - rlo).abs().max() < 1e-5 and (hi.cpu() - rhi).abs().max() < 1e-5
    bad = torch.zeros(C + 1)
    bad[C] = 1
    with pytest.raises(_lib.IrnError, match="out of range"):
        cam_ops.merge_cams([o[:C].to(cuda_dev) for o in outs], (H, W), bad)


def test_irn_crop640_vs_fp64_oracle_and_ragged_bitwise(cuda_dev, images):
    sd = synth.irn_state_dict()
    m = EdgeDisplacement(crop_size=640)
    m.load_state_dict(sd, strict=False)
    sd64 = _sd64(sd, cuda_dev)
    sizes = [SIZES[0], SIZES[2]]
    ims = [images[0], images[2]]
    edge_r, dp_r = m.forward_ragged([im for im in ims])
    assert edge_r.shape == (2, 1, 160, 160)
    for i, im in enumerate(ims):
        x = preprocess.resize_normalize(im, im.shape[:2])
        e, d = m(x)
        re, rd = nets.edge_displacement(x.double(), sd64, crop_size=640)
        assert float((e.double() - re).abs().max()) < 1e-4 and float((d.double() - rd).abs().max()) < 1e-4
        fh, fw = e.shape[-2:]
        assert torch.equal(edge_r[i, :, :fh, :fw], e) and torch.equal(dp_r[i, :, :fh, :fw], d)
    with pytest.raises(_lib.IrnError):
        EdgeDisplacement().forward_ragged([ims[0]])


def test_walk_160_vs_fp64_oracle_and_padded_bitwise(cuda_dev):
    h = w = 160
    e = synth.edge_map(h, w, "bimodal", 3)
    x = synth.seeds(2, h, w, 3)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_dev)
    out = indexing.random_walk_batch(t(x), t(e), [0, 2], 5, 10, 256).cpu().numpy()
    assert not indexing.last_walk_was_fused()        # the per-step kernel walks grids beyond 128 x 128
    truth = oi.propagate_stencil(x, e, 5, 10, 256).reshape(2, h, w)
    assert np.abs(out - truth).max() < 2e-6
    # a 600 x 500 image on the 640 crop: feature grid 150 x 125 inside the 160 x 160 pad, edge 1 outside
    fh, fw = 150, 125
    ep = np.ones((1, h, w), np.float32)
    ep[:, :fh, :fw] = e[:, :fh, :fw]
    for exp_times in (0, 8):
        pipe = PseudoLabelPipeline(None, None, cuda_dev, exp_times=exp_times)
        own, _ = pipe.walk_stage([t(x[:, :fh, :fw])], t(e[:, :fh, :fw]))
        pad = pipe.walk_padded_stage([t(x[:, :fh, :fw])], t(ep), [(600, 500)])
        assert torch.equal(pad[0], own), exp_times


def _oracle_q(img, lab, n):
    d = ocrf.DenseCRF2D(img.shape[1], img.shape[0], n)
    d.setUnaryEnergy(ocrf.unary_from_labels(lab, n, 0.7))
    d.addPairwiseGaussian(sxy=3, compat=3)
    d.addPairwiseBilateral(sxy=50, srgb=5, rgbim=img, compat=10)
    return d.inference(10).reshape(n, *img.shape[:2]), [p.lattice.n_vertices for p in d.pairwise]


@pytest.mark.parametrize("n", [22, 33, 64, 81])
def test_crf_many_labels_bitwise(cuda_dev, n):
    from irn_b200 import crf
    assert crf.max_labels() >= 81
    H, W = 24, 32
    img = synth.image(n, H, W)
    lab = np.random.RandomState(n).randint(0, n, (H, W)).astype(np.int32)
    q_ref, counts_ref = _oracle_q(img, lab, n)
    labels, q, counts = crf.dense_crf(torch.from_numpy(img)[None].to(cuda_dev), torch.from_numpy(lab)[None].to(cuda_dev), n, want_q=True)
    assert counts[0].tolist() == counts_ref
    assert np.array_equal(q[0].cpu().numpy(), q_ref)
    assert np.array_equal(labels[0].cpu().numpy(), np.argmax(q_ref, 0))


def test_ir_label_30_classes(cuda_dev):
    from irn_b200 import crf
    H, W = 60, 80
    img = synth.image(30, H, W)
    keys = np.sort(np.random.RandomState(1).choice(C, 30, replace=False))
    high = synth.u8_to_cam(synth.cam_planes_u8(30, H, W, 2))
    conf = crf.ir_labels(torch.from_numpy(img)[None].to(cuda_dev), [high], [keys], 0.30, 0.05, n_classes=C)[0].cpu().numpy()
    ref = ocrf.cam_to_ir_label_one(img, high, keys)["conf"]
    assert np.array_equal(conf, ref)
    assert conf.max() > 20          # class ids beyond VOC's reach the map


# ------------------------------------------------------------------------------------------------ steps on a synthetic COCO tree
TREE_SIZES = [(640, 480), (480, 640), (427, 640), (640, 640), (375, 500), (333, 500), (480, 640), (427, 640)]


@pytest.fixture(scope="module")
def coco_tree(tmp_path_factory, cuda_dev):
    root = tmp_path_factory.mktemp("coco")
    os.makedirs(root / "train2014")
    os.makedirs(root / "gt")
    os.makedirs(root / "sess")
    stems, labels = [], {}
    for i, (h, w) in enumerate(TREE_SIZES):
        stem = "train2014/COCO_train2014_%012d" % (100 + i)
        img = synth.image(900 + i, h, w)
        if i == 5:
            Image.fromarray(img[..., 1]).save(root / (stem + ".jpg"), quality=92)     # greyscale
        else:
            Image.fromarray(img).save(root / (stem + ".jpg"), quality=92)
        labels[stem] = synth.label(i, n_classes=C)
        gt = np.zeros((h, w), np.uint8)
        gt[h // 4:3 * h // 4, w // 4:3 * w // 4] = 1 + int(np.flatnonzero(labels[stem])[0])
        gt[:2] = 255
        Image.fromarray(gt).save(root / "gt" / (os.path.basename(stem) + ".png"))
        stems.append(stem)
    np.save(root / "cls_labels.npy", labels)
    (root / "list.txt").write_text("\n".join(stems) + "\n")
    torch.save(synth.cam_state_dict(seed=5, n_classes=C), root / "sess" / "cam80.pth.pth")
    torch.save(synth.irn_state_dict(), root / "sess" / "irn.pth")
    return root, stems


def _args(root, out, **kw):
    a = dict(num_workers=0, dataset="coco", coco_root=str(root), coco_cls_labels=str(root / "cls_labels.npy"), coco_gt_dir=str(root / "gt"),
             train_list=str(root / "list.txt"), infer_list=str(root / "list.txt"), cam_network="irn_b200.cam", irn_network="irn_b200.irn",
             cam_scales=SCALES, cam_weights_name=str(root / "sess" / "cam80.pth"), irn_weights_name=str(root / "sess" / "irn.pth"),
             irn_crop_size=640, beta=10, exp_times=8, sem_seg_bg_thres=0.25, ins_seg_bg_thres=0.25, conf_fg_thres=0.30,
             conf_bg_thres=0.05, cam_eval_thres=0.15, synthetic=0, step_batch=4, device_pyramid=True, device_jpeg=False)
    a.update(kw)
    for d in ("cam", "ir_label", "sem_seg", "ins_seg"):
        os.makedirs(out / d, exist_ok=True)
        a[d + "_out_dir"] = str(out / d)
    return types.SimpleNamespace(**a)


def _run_all(args):
    from irn_b200.step import cam_to_ir_label, make_cam, make_ins_seg_labels, make_sem_seg_labels
    make_cam.run(args)
    cam_to_ir_label.run(args)
    make_ins_seg_labels.run(args)
    make_sem_seg_labels.run(args)


def _same_outputs(a, b, names):
    for n in names:
        da = np.load(os.path.join(a.cam_out_dir, n + ".npy"), allow_pickle=True).item()
        db = np.load(os.path.join(b.cam_out_dir, n + ".npy"), allow_pickle=True).item()
        assert np.array_equal(np.asarray(da["keys"]), np.asarray(db["keys"])), n
        assert np.array_equal(np.asarray(da["cam"]), np.asarray(db["cam"])) and np.array_equal(da["high_res"], db["high_res"]), n
        for d in ("ir_label_out_dir", "sem_seg_out_dir"):
            pa = np.asarray(Image.open(os.path.join(getattr(a, d), n + ".png")))
            assert np.array_equal(pa, np.asarray(Image.open(os.path.join(getattr(b, d), n + ".png")))), (d, n)
        # byte for byte: a detection whose walk is all zero scores NaN (0 / 0, as in the reference), and NaN != NaN
        ia = np.load(os.path.join(a.ins_seg_out_dir, n + ".npy"), allow_pickle=True).item()
        ib = np.load(os.path.join(b.ins_seg_out_dir, n + ".npy"), allow_pickle=True).item()
        assert sorted(ia) == sorted(ib), n
        for k in ia:
            va, vb = np.asarray(ia[k]), np.asarray(ib[k])
            assert va.dtype == vb.dtype and va.shape == vb.shape and va.tobytes() == vb.tobytes(), (n, k)


def test_steps_on_synthetic_coco(coco_tree, tmp_path):
    root, stems = coco_tree
    names = [os.path.basename(s) for s in stems]
    batched = _args(root, tmp_path / "batched")
    _run_all(batched)
    labels = np.load(root / "cls_labels.npy", allow_pickle=True).item()
    for stem, n in zip(stems, names):
        d = np.load(os.path.join(batched.cam_out_dir, n + ".npy"), allow_pickle=True).item()
        assert np.array_equal(d["keys"].numpy(), np.flatnonzero(labels[stem]))
        H, W = Image.open(root / (stem + ".jpg")).size[::-1]
        assert d["high_res"].shape == (len(d["keys"]), H, W)
        sem = np.asarray(Image.open(os.path.join(batched.sem_seg_out_dir, n + ".png")))
        assert sem.shape == (H, W) and set(np.unique(sem)) <= {0} | set(int(k) + 1 for k in d["keys"])
    one = _args(root, tmp_path / "one", step_batch=1)
    _run_all(one)
    _same_outputs(batched, one, names)
    dev = _args(root, tmp_path / "dev", device_jpeg=True)
    _run_all(dev)
    _same_outputs(batched, dev, names)

    # evaluation over 81 classes against a numpy confusion of the same files
    from irn_b200.step import eval_cam, eval_sem_seg
    gts = []
    for n in names:
        g = np.asarray(Image.open(root / "gt" / (n + ".png"))).astype(np.int64)
        g[g == 255] = -1
        gts.append(g)

    def miou(preds):
        conf = np.zeros((81, 81), np.int64)
        for p, g in zip(preds, gts):
            ok = g >= 0
            np.add.at(conf, (g[ok], p[ok].astype(np.int64)), 1)
        with np.errstate(divide="ignore", invalid="ignore"):
            iou = np.diag(conf) / (conf.sum(0) + conf.sum(1) - np.diag(conf))
        return np.nanmean(iou)
    cam_preds = []
    for n in names:
        d = np.load(os.path.join(batched.cam_out_dir, n + ".npy"), allow_pickle=True).item()
        cams = np.concatenate([np.full((1,) + d["high_res"].shape[1:], 0.15, np.float32), d["high_res"]])
        cam_preds.append(np.concatenate([[0], np.asarray(d["keys"]) + 1])[np.argmax(cams, 0)])
    assert np.isclose(eval_cam.run(batched)["miou"], miou(cam_preds), rtol=0, atol=1e-12)
    sem_preds = []
    for n in names:
        p = np.asarray(Image.open(os.path.join(batched.sem_seg_out_dir, n + ".png"))).copy()
        p[p == 255] = 0
        sem_preds.append(p)
    assert np.isclose(eval_sem_seg.run(batched)["miou"], miou(sem_preds), rtol=0, atol=1e-12)


def test_ir_labels_class_count(cuda_dev):
    """cam_to_ir_label's CRF takes background + up to 128 classes (129 labels); ir_labels holds an image's class ids to the
    dataset's class count (20 by default, PASCAL VOC's; 80 for MS COCO)."""
    from irn_b200 import crf
    assert crf.max_labels() == 129
    img = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device=cuda_dev)

    def run(K, n_classes, keys=None):
        keys = np.arange(K) if keys is None else np.asarray(keys)
        return crf.ir_labels(img, [np.zeros((K, 8, 8), np.float32)], [keys], 0.3, 0.05, n_classes=n_classes)
    for K, n in ((40, 20), (21, 20), (81, 80), (1, 0), (1, 129)):
        with pytest.raises(_lib.IrnError):
            run(K, n)
    with pytest.raises(_lib.IrnError, match="class id 20"):
        run(2, 20, keys=[3, 20])
    with pytest.raises(_lib.IrnError, match="class id 80"):
        run(1, 80, keys=[80])
    for K, n in ((20, 20), (40, 80), (80, 80), (128, 128)):
        assert run(K, n).shape == (1, 8, 8)
