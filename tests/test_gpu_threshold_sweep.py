"""The background-threshold sweep on the GPU (indexing.ThresholdSweep, step.sweep_cam, step.sweep_sem_seg).

  planes   eval_cam's high_res used as stored: device confusions equal oracle/threshold_sweep.py bit for bit, at 375x500, 500x375,
           640x640, 1x1, 1xW and Hx1, K = 0, 1, 3, 20 and 80, thresholds placed on pixel values, NaN planes
  walk     for every threshold the confusion of the existing rw_labels maps, C up to 80 and an all-zero walk (0/0: keys[0] + 1)
  steps    on a synthetic VOC tree and a synthetic 80-class COCO tree: sweep_cam row j is eval_cam at t_j; sweep_sem_seg at three
           thresholds is make_sem_seg_labels + eval_sem_seg at each; --step_batch 1 and 4 agree
  streams  late inputs released on a side stream give the default-stream result
  errors   a label >= n_class, a size mismatch, T = 257 and non-ascending thresholds raise IrnError; the device stays usable
  spawn    with >= 2 GPUs the spawn branch of sweep_sem_seg equals one GPU
"""
import os
import types

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import golden_path
from irn_b200 import _lib, indexing, synth
from irn_b200.step import _voc_eval
from oracle import threshold_sweep

pytestmark = pytest.mark.gpu


def _planes(rs, K, H, W, n_vals=None):
    s = rs.uniform(0, 1, (K, H, W)).astype(np.float32)
    if n_vals:      # few distinct values: ties between planes and with the thresholds
        s = np.round(s * n_vals) / n_vals
    return s.astype(np.float32)


PLANE_CASES = [((375, 500), 3), ((500, 375), 20), ((640, 640), 80), ((1, 1), 1), ((1, 333), 3), ((257, 1), 20), ((375, 500), 0),
               ((64, 48), 1)]


def test_planes_vs_oracle(cuda_dev):
    rs = np.random.RandomState(0)
    for n_class in (21, 81):
        scores, keys, gts = [], [], []
        for (H, W), K in PLANE_CASES:
            if K >= n_class:
                continue
            s = _planes(rs, K, H, W, n_vals=16 if K % 2 else None)
            if K == 20:
                s[3][rs.rand(H, W) < 0.05] = np.nan
            scores.append(s)
            keys.append(np.sort(rs.choice(n_class - 1, K, replace=False)))
            g = rs.randint(0, n_class, (H, W)).astype(np.uint8)
            g[rs.rand(H, W) < 0.1] = 255
            gts.append(g)
        vals = np.concatenate([s.reshape(-1) for s in scores if s.size])
        vals = vals[np.isfinite(vals)]
        for T in (1, 91, 256):
            thr = np.unique(np.concatenate([rs.choice(vals, T // 2 + 1), rs.uniform(0, 1, T).astype(np.float32)]))[:T]
            sweep = indexing.ThresholdSweep(thr, n_class, cuda_dev)
            assert np.array_equal(sweep.thresholds, thr)
            for s, k, g in zip(scores, keys, gts):
                sweep.add_cam(torch.from_numpy(s).to(cuda_dev), k, torch.from_numpy(g).to(cuda_dev))
            ref = threshold_sweep.sweep_confusion(scores, keys, [np.where(g == 255, -1, g.astype(np.int64)) for g in gts], thr, n_class)
            got = sweep.confusion()
            assert got.dtype == np.int64 and np.array_equal(got, ref), (n_class, T, int((got != ref).sum()))


def _walk_case(rs, C, h, w, zero=False):
    rw = np.zeros((C, h, w), np.float32) if zero else rs.uniform(0, 1, (C, h, w)).astype(np.float32) ** 3
    return rw


@pytest.mark.parametrize("C,h,w,H,W,zero", [(1, 24, 28, 94, 111, False), (3, 94, 125, 375, 500, False), (20, 160, 160, 640, 640, False),
                                            (80, 40, 30, 160, 118, False), (2, 20, 20, 80, 77, True)])
def test_walk_vs_rw_labels(cuda_dev, C, h, w, H, W, zero):
    rs = np.random.RandomState(C + h)
    n_class = 81 if C >= 20 else 21
    rw = torch.from_numpy(_walk_case(rs, C, h, w, zero)).to(cuda_dev)
    keys = np.sort(rs.choice(n_class - 1, C, replace=False))
    g = rs.randint(0, n_class, (H, W)).astype(np.uint8)
    g[rs.rand(H, W) < 0.1] = 255
    _, _, up = indexing.rw_labels(rw, keys, (H, W), 0.25, want_scores=True)
    vals = up.cpu().numpy().reshape(-1)
    vals = vals[np.isfinite(vals)] if not zero else np.float32([0.5])
    thr = np.unique(np.concatenate([rs.choice(vals, 6), np.float32([0.05, 0.25, 0.5, 0.95])]))
    sweep = indexing.ThresholdSweep(thr, n_class, cuda_dev)
    sweep.add_walk(rw[:, None], keys, (H, W), torch.from_numpy(g).to(cuda_dev))
    got = sweep.confusion()
    gt = np.where(g == 255, -1, g.astype(np.int64))
    for j, t in enumerate(sweep.thresholds):
        lab, _, _ = indexing.rw_labels(rw, keys, (H, W), float(t))
        lab = lab.cpu().numpy()
        if zero:
            assert (lab == keys[0] + 1).all()
        assert np.array_equal(got[j], _voc_eval.confusion([lab], [gt], n_class)), (j, float(t))


def test_walk_without_classes_is_background(cuda_dev):
    """The zero fill of label_ragged_stage: a walk of no channels is background at every threshold."""
    g = torch.randint(0, 21, (37, 41), dtype=torch.uint8, device=cuda_dev)
    sweep = indexing.ThresholdSweep([0.1, 0.5], 21, cuda_dev)
    sweep.add_walk(torch.zeros((0, 10, 11), device=cuda_dev), [], (37, 41), g)
    conf = sweep.confusion()
    want = np.bincount(g.cpu().numpy().reshape(-1).astype(np.int64), minlength=21)
    assert np.array_equal(conf[:, :, 0], np.stack([want, want])) and not conf[:, :, 1:].any()


def test_late_inputs_on_side_stream(cuda_dev):
    rs = np.random.RandomState(3)
    s = torch.from_numpy(_planes(rs, 3, 200, 300, 8)).to(cuda_dev)
    rw = torch.from_numpy(_walk_case(rs, 2, 50, 75)).to(cuda_dev)
    g = torch.from_numpy(rs.randint(0, 21, (200, 300)).astype(np.uint8)).to(cuda_dev)
    thr = np.linspace(0.05, 0.95, 91)

    def run(sc, w, gt):
        sw = indexing.ThresholdSweep(thr, 21, cuda_dev)
        sw.add_cam(sc, [2, 5, 9], gt)
        sw.add_walk(w, [4, 7], (200, 300), gt)
        return sw.confusion()
    want = run(s, rw, g)
    side = torch.cuda.Stream(cuda_dev)
    side.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(side):
        bufs = [torch.full_like(s, float("nan")), torch.full_like(rw, 7.0), torch.full_like(g, 250)]
        torch.cuda._sleep(20_000_000)
        for b, src in zip(bufs, (s, rw, g)):
            b.copy_(src)
        got = run(*bufs)
    assert np.array_equal(got, want)


def test_errors_raise_without_fault(cuda_dev):
    g = torch.zeros((8, 8), dtype=torch.uint8, device=cuda_dev)
    s = torch.ones((1, 8, 8), device=cuda_dev)
    sw = indexing.ThresholdSweep([0.5], 21, cuda_dev)
    sw.add_cam(s, [25], g)                          # label 26 >= 21
    with pytest.raises(_lib.IrnError, match="predicted label 26"):
        sw.confusion()
    sw = indexing.ThresholdSweep([0.5], 21, cuda_dev)
    sw.add_cam(s, [2], torch.full((8, 8), 40, dtype=torch.uint8, device=cuda_dev))
    with pytest.raises(_lib.IrnError, match="ground-truth label 40"):
        sw.confusion()
    with pytest.raises(_lib.IrnError, match="ground truth must be"):
        sw.add_cam(s, [2], torch.zeros((8, 9), dtype=torch.uint8, device=cuda_dev))
    with pytest.raises(_lib.IrnError, match="keys"):
        sw.add_cam(s, [2, 3], g)
    with pytest.raises(_lib.IrnError, match="257"):
        indexing.ThresholdSweep(np.linspace(0, 1, 257), 21, cuda_dev)
    L = _lib.lib()
    keys = np.array([0, 3], np.int32)
    thr = np.float32([0.5, 0.4])
    hist = torch.zeros(L.irn_threshold_sweep_bytes(2, 21), dtype=torch.uint8, device=cuda_dev)
    rc = L.irn_threshold_sweep_accumulate(0, _lib.ptr(s), 1, 8, 8, 8, 8, keys.ctypes.data, _lib.ptr(g), thr.ctypes.data, 2, 21,
                                          _lib.ptr(hist), None, _lib.stream_ptr())
    assert rc == -1 and b"ascending" in L.irn_last_error()
    torch.cuda.synchronize()
    sw = indexing.ThresholdSweep([0.5], 21, cuda_dev)        # the device is still usable
    sw.add_cam(s, [2], g)
    assert sw.confusion()[0, 0, 3] == 64


# ------------------------------------------------------------------------------------------------------------------------- steps
def _gt_png(path, arr):
    im = Image.new("P", (arr.shape[1], arr.shape[0]))
    im.putdata(arr.reshape(-1).tolist())
    im.putpalette([v for k in range(256) for v in (k, k, k)])
    im.save(path)


@pytest.fixture(scope="module")
def voc_tree(tmp_path_factory, cuda_dev):
    """The three images of tests/golden/steps.npz as a VOC tree with seeded ground truth, and make_cam's CAMs."""
    g = np.load(golden_path("steps.npz"))
    root = tmp_path_factory.mktemp("voc_sweep")
    for d in ("JPEGImages", "SegmentationClass", "ImageSets/Segmentation", "sess", "cam"):
        os.makedirs(root / d)
    ids = [str(s) for s in g["ids"]]
    labels = {}
    rs = np.random.RandomState(9)
    for i, name in enumerate(ids):
        img = g["img%d" % i]
        Image.fromarray(img).save(root / "JPEGImages" / (name + ".jpg"), format="PNG")
        labels[int(name.replace("_", ""))] = g["label%d" % i]
        H, W = img.shape[:2]
        gt = np.zeros((H, W), np.uint8)
        cls = np.flatnonzero(g["label%d" % i])
        gt[H // 4:3 * H // 4, W // 4:3 * W // 4] = cls[0] + 1
        gt[rs.rand(H, W) < 0.05] = 255
        _gt_png(root / "SegmentationClass" / (name + ".png"), gt)
    np.save(root / "cls_labels.npy", labels, allow_pickle=True)
    (root / "list.txt").write_text("\n".join(ids) + "\n")
    (root / "ImageSets" / "Segmentation" / "train.txt").write_text("\n".join(ids) + "\n")
    torch.save(synth.cam_state_dict(), root / "sess" / "res50_cam.pth.pth")
    torch.save(synth.irn_state_dict(), root / "sess" / "res50_irn.pth")
    args = types.SimpleNamespace(
        num_workers=0, voc12_root=str(root), train_list=str(root / "list.txt"), infer_list=str(root / "list.txt"), chainer_eval_set="train",
        cam_network="irn_b200.cam", irn_network="irn_b200.irn", cam_scales=(1.0, 0.5, 1.5, 2.0),
        cam_weights_name=str(root / "sess" / "res50_cam.pth"), irn_weights_name=str(root / "sess" / "res50_irn.pth"),
        cam_out_dir=str(root / "cam"), beta=10, exp_times=8, sem_seg_bg_thres=0.25, cam_eval_thres=0.15, synthetic=0, step_batch=4)
    from irn_b200.voc12 import dataloader
    dataloader._cls_labels["voc12/cls_labels.npy"] = labels
    from irn_b200.step import make_cam
    make_cam.run(args)
    return root, ids, args


@pytest.fixture(scope="module")
def coco_tree(tmp_path_factory, cuda_dev):
    """Eight synthetic MS COCO images up to 640 pixels over 80 classes, class-index ground truth, and make_cam's CAMs."""
    sizes = [(640, 480), (480, 640), (427, 640), (640, 640), (375, 500), (333, 500), (480, 640), (427, 640)]
    root = tmp_path_factory.mktemp("coco_sweep")
    for d in ("train2014", "gt", "sess", "cam"):
        os.makedirs(root / d)
    stems, labels = [], {}
    rs = np.random.RandomState(11)
    for i, (h, w) in enumerate(sizes):
        stem = "train2014/COCO_train2014_%012d" % (300 + i)
        Image.fromarray(synth.image(950 + i, h, w)).save(root / (stem + ".jpg"), quality=92)
        labels[stem] = synth.label(i, n_classes=80)
        gt = np.zeros((h, w), np.uint8)
        cls = np.flatnonzero(labels[stem])
        gt[h // 4:3 * h // 4, w // 4:3 * w // 4] = 1 + int(cls[0])
        gt[:h // 8, :w // 8] = 1 + int(cls[-1])
        gt[rs.rand(h, w) < 0.02] = 255
        Image.fromarray(gt).save(root / "gt" / (os.path.basename(stem) + ".png"))
        stems.append(stem)
    np.save(root / "cls_labels.npy", labels)
    (root / "list.txt").write_text("\n".join(stems) + "\n")
    torch.save(synth.cam_state_dict(seed=5, n_classes=80), root / "sess" / "cam80.pth.pth")
    torch.save(synth.irn_state_dict(), root / "sess" / "irn.pth")
    args = types.SimpleNamespace(
        num_workers=0, dataset="coco", coco_root=str(root), coco_cls_labels=str(root / "cls_labels.npy"), coco_gt_dir=str(root / "gt"),
        train_list=str(root / "list.txt"), infer_list=str(root / "list.txt"), cam_network="irn_b200.cam", irn_network="irn_b200.irn",
        cam_scales=(1.0, 0.5, 1.5, 2.0), cam_weights_name=str(root / "sess" / "cam80.pth"), irn_weights_name=str(root / "sess" / "irn.pth"),
        irn_crop_size=640, beta=10, exp_times=8, sem_seg_bg_thres=0.25, cam_eval_thres=0.15, synthetic=0, step_batch=4,
        device_pyramid=True, device_jpeg=False, cam_out_dir=str(root / "cam"))
    from irn_b200.step import make_cam
    make_cam.run(args)
    return root, [os.path.basename(s) for s in stems], args


TREES = ["voc_tree", "coco_tree"]


def _with(args, **kw):
    a = types.SimpleNamespace(**vars(args))
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _same_scores(got, want, what):
    assert got.shape == want.shape and got.tobytes() == want.tobytes(), what     # bitwise, NaN where eval leaves NaN


@pytest.mark.parametrize("tree", TREES)
def test_sweep_cam_rows_equal_eval_cam(request, tree):
    _, _, args = request.getfixturevalue(tree)
    from irn_b200.step import eval_cam, sweep_cam
    thr = [0.05, 0.1, 0.15, 0.2, 0.3, 0.5, 0.8, 0.95]
    out = sweep_cam.run(_with(args, cam_eval_thres_sweep=",".join(map(str, thr[::-1]))))
    assert np.array_equal(out["thresholds"], np.float32(thr)) and out["iou"].shape[0] == len(thr)
    for j, t in enumerate(thr):
        ref = eval_cam.run(_with(args, cam_eval_thres=t))
        _same_scores(out["iou"][j], np.asarray(ref["iou"], np.float64), (tree, t))
        assert out["miou"][j] == ref["miou"] or (np.isnan(out["miou"][j]) and np.isnan(ref["miou"]))
    assert out["best"] == float(out["thresholds"][int(np.nanargmax(out["miou"]))])
    b1 = sweep_cam.run(_with(args, cam_eval_thres_sweep=thr, step_batch=1))
    assert b1["iou"].tobytes() == out["iou"].tobytes()


@pytest.mark.parametrize("tree", TREES)
def test_sweep_sem_seg_equals_make_and_eval(request, tree, tmp_path):
    _, _, args = request.getfixturevalue(tree)
    from irn_b200.step import eval_sem_seg, make_sem_seg_labels, sweep_sem_seg
    thr = [0.15, 0.25, 0.6]
    out = {}
    for bsz in (4, 1):
        out[bsz] = sweep_sem_seg.run(_with(args, sem_seg_bg_thres_sweep=thr, step_batch=bsz))
    assert out[4]["iou"].tobytes() == out[1]["iou"].tobytes()
    for j, t in enumerate(thr):
        d = tmp_path / ("sem%d" % j)
        os.makedirs(d)
        a = _with(args, sem_seg_bg_thres=t, sem_seg_out_dir=str(d))
        make_sem_seg_labels.run(a)
        ref = eval_sem_seg.run(a)
        _same_scores(out[4]["iou"][j], np.asarray(ref["iou"], np.float64), (tree, t))


def test_missing_cam_names_the_image(voc_tree, tmp_path):
    root, ids, args = voc_tree
    from irn_b200.step import sweep_cam, sweep_sem_seg
    d = tmp_path / "cam"
    os.makedirs(d)
    for i in ids[:-1]:
        os.symlink(os.path.join(args.cam_out_dir, i + ".npy"), d / (i + ".npy"))
    for step in (sweep_cam, sweep_sem_seg):
        with pytest.raises(FileNotFoundError, match=ids[-1]):
            step.run(_with(args, cam_out_dir=str(d)))


_SPAWN_CHILD = """
import sys, pickle
sys.path.insert(0, {root!r})
from irn_b200.voc12 import dataloader
from irn_b200.step import sweep_sem_seg
args = pickle.load(open({args!r}, 'rb'))
dataloader._cls_labels["voc12/cls_labels.npy"] = pickle.load(open({labels!r}, 'rb'))
out = sweep_sem_seg.run(args)
pickle.dump(out, open({out!r}, 'wb'))
"""


def test_spawn_branch_matches_single_gpu(voc_tree, tmp_path):
    import pickle
    import subprocess
    import sys
    from conftest import ROOT
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root, _, args = voc_tree
    from irn_b200.voc12 import dataloader
    pickle.dump(_with(args, sem_seg_bg_thres_sweep=[0.1, 0.25, 0.5], step_batch=2), open(tmp_path / "args.pkl", "wb"))
    pickle.dump(dataloader._cls_labels["voc12/cls_labels.npy"], open(tmp_path / "labels.pkl", "wb"))
    res = {}
    for tag, visible in (("multi", None), ("single", "0")):
        env = dict(os.environ, PYTHONPATH=ROOT)
        if visible is not None:
            env["CUDA_VISIBLE_DEVICES"] = visible
        code = _SPAWN_CHILD.format(root=ROOT, args=str(tmp_path / "args.pkl"), labels=str(tmp_path / "labels.pkl"),
                                   out=str(tmp_path / (tag + ".pkl")))
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900, cwd=str(tmp_path))
        assert r.returncode == 0, r.stderr[-3000:]
        res[tag] = pickle.load(open(tmp_path / (tag + ".pkl"), "rb"))
    assert res["multi"]["iou"].tobytes() == res["single"]["iou"].tobytes()
