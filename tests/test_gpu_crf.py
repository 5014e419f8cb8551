"""The device CRF (irn_b200.crf, irn_b200/csrc/crf.cu) against the oracle (oracle/crf.py) and against the cam_to_ir_label fixture
(tests/golden/ir_label.npz: the unmodified reference's step with the oracle as its pydensecrf); the step end to end."""
import hashlib
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import ROOT, golden_path, record
from irn_b200 import synth
from oracle import crf as ocrf

pytestmark = pytest.mark.gpu

G = np.load(golden_path("ir_label.npz"))
STEPS = np.load(golden_path("steps.npz"))


def _case(i):
    if ("seed%d" % i) in G:
        H, W = G["png%d" % i].shape
        keys = G["keys%d" % i]
        u8 = synth.cam_planes_u8(len(keys), H, W, int(G["seed%d" % i]))
        assert hashlib.sha256(np.ascontiguousarray(u8).tobytes()).hexdigest() == str(G["cam_sha256%d" % i]), \
            "synth.cam_planes_u8 no longer regenerates the fixture's CAM planes"
        return synth.image(int(G["seed%d" % i]), H, W), synth.u8_to_cam(u8)
    j = int(G["steps_index%d" % i])
    return STEPS["img%d" % j], STEPS["cam_high%d" % j].astype(np.float32)


def _oracle_q(img, lab, n, t, gt, gauss, bil):
    d = ocrf.DenseCRF2D(img.shape[1], img.shape[0], n)
    d.setUnaryEnergy(ocrf.unary_from_labels(lab, n, gt))
    d.addPairwiseGaussian(sxy=gauss[0], compat=gauss[1])
    d.addPairwiseBilateral(sxy=bil[0], srgb=bil[1], rgbim=img, compat=bil[2])
    counts = [p.lattice.n_vertices for p in d.pairwise]
    return d.inference(t).reshape(n, *img.shape[:2]), counts


# (H, W, n_labels, t, gt_prob, gauss (sxy, compat), bilateral (sxy, srgb, compat), seed)
Q_CASES = [
    (1, 1, 2, 10, 0.7, (3, 3), (50, 5, 10), 0),
    (3, 5, 3, 1, 0.7, (3, 3), (50, 5, 10), 1),
    (3, 5, 1, 10, 0.7, (3, 3), (50, 5, 10), 2),
    (20, 24, 5, 0, 0.9, (3, 3), (50, 5, 10), 3),
    (20, 24, 5, 1, 0.9, (2, 5), (30, 8, 4), 3),
    (20, 24, 5, 10, 0.7, (2, 5), (30, 8, 4), 3),
    (375, 500, 2, 10, 0.7, (3, 3), (50, 5, 10), 4),
    (500, 375, 3, 1, 0.9, (3, 3), (50, 5, 10), 5),
    (512, 512, 21, 10, 0.7, (3, 3), (50, 5, 10), 6),
]


@pytest.mark.parametrize("case", Q_CASES, ids=lambda c: "%dx%d_n%d_t%d" % c[:4])
def test_q_and_vertex_counts_match_oracle(cuda_dev, case):
    from irn_b200 import crf
    H, W, n, t, gt, gauss, bil, seed = case
    img = synth.image(seed, H, W) if H * W > 1 else np.array([[[10, 20, 30]]], np.uint8)
    rs = np.random.RandomState(seed)
    lab = (synth.cam_planes_u8(n, H, W, seed).argmax(0) if H * W > 64 and n > 1 else rs.randint(0, n, (H, W))).astype(np.int32)
    q_ref, counts_ref = _oracle_q(img, lab, n, t, gt, gauss, bil)
    labels, q, counts = crf.dense_crf(torch.from_numpy(img)[None].to(cuda_dev), torch.from_numpy(lab)[None].to(cuda_dev), n, t=t,
                                      gt_prob=gt, gauss=gauss, bilateral=bil, want_q=True)
    assert counts[0].tolist() == counts_ref
    q = q[0].cpu().numpy()
    err = float(np.abs(q - q_ref).max())
    flips = float((labels[0].cpu().numpy() != np.argmax(q_ref, 0)).mean())
    record("crf_q_%dx%d_n%d_t%d" % (H, W, n, t), q_max_abs=err, label_disagreement=flips, vertices_bilateral=counts[0][1])
    assert err < 1e-5
    assert flips <= 1e-3


def test_batch_with_mixed_content_and_determinism(cuda_dev):
    """A batch gives what each image gives alone, and two identical calls are bitwise equal."""
    from irn_b200 import crf
    imgs = np.stack([synth.image(20 + i, 64, 80) for i in range(3)])
    labs = np.stack([synth.cam_planes_u8(4, 64, 80, i).argmax(0) for i in range(3)]).astype(np.int32)
    x, l = torch.from_numpy(imgs).to(cuda_dev), torch.from_numpy(labs).to(cuda_dev)
    a = crf.dense_crf(x, l, 4, want_q=True)
    b = crf.dense_crf(x, l, 4, want_q=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    for i in range(3):
        s = crf.dense_crf(x[i:i + 1], l[i:i + 1], 4, want_q=True)
        assert torch.equal(s[1][0], a[1][i]) and s[2][0].tolist() == a[2][i].tolist()


def test_crf_inference_label_matches_oracle(cuda_dev):
    from irn_b200.misc import imutils
    img, high = _case(0)
    lab = G["fg_conf_cam0"].astype(np.int64)
    n = len(G["keys0"]) + 1
    got = imutils.crf_inference_label(img, lab, n_labels=n)
    assert got.shape == lab.shape
    assert (got != G["pred_fg0"]).mean() <= 1e-3
    assert (imutils.crf_inference_label(img, np.zeros_like(lab), n_labels=1) == 0).all()


def test_ir_labels_match_fixture(cuda_dev):
    """irn_ir_label per fixture case and as one batch per image size: conf maps within 0.1 % of the reference's PNGs, 0 and 255
    only where the fixture has them, identical batched and alone."""
    from irn_b200 import crf
    n = int(G["n"])
    by_size = {}
    for i in range(n):
        img, high = _case(i)
        x = torch.from_numpy(img)[None].to(cuda_dev)
        conf, vc = crf.ir_labels(x, [high], [G["keys%d" % i]], float(G["conf_fg_thres"]), float(G["conf_bg_thres"]),
                                 return_counts=True)
        conf = conf[0].cpu().numpy()
        ref = G["png%d" % i]
        bad = float((conf != ref).mean())
        record("ir_label_fixture_%d" % i, disagreement=bad, vertices_gauss=vc[0][0], vertices_bilateral=vc[0][1])
        assert bad <= 1e-3
        for v in (0, 255):
            assert not ((conf == v) & (ref != v) & (conf != ref)).sum() > 1e-3 * ref.size
        by_size.setdefault(img.shape, []).append((i, img, high, conf))
    for items in by_size.values():
        if len(items) < 2:
            continue
        x = torch.from_numpy(np.stack([it[1] for it in items])).to(cuda_dev)
        conf = crf.ir_labels(x, [it[2] for it in items], [G["keys%d" % it[0]] for it in items], 0.30, 0.05).cpu().numpy()
        for k, it in enumerate(items):
            assert np.array_equal(conf[k], it[3])


def test_errors(cuda_dev):
    from irn_b200 import crf, _lib
    img = torch.zeros(1, 8, 8, 3, dtype=torch.uint8)
    lab = torch.zeros(1, 8, 8, dtype=torch.int32)
    with pytest.raises(_lib.IrnError):
        crf.dense_crf(img, lab.to(cuda_dev), 2)
    with pytest.raises(_lib.IrnError):
        crf.dense_crf(img.to(cuda_dev), lab, 2)
    bad = lab.clone()
    bad[0, 3, 3] = 2
    with pytest.raises(_lib.IrnError, match="outside"):
        crf.dense_crf(img.to(cuda_dev), bad.to(cuda_dev), 2)
    bad[0, 3, 3] = -1
    with pytest.raises(_lib.IrnError, match="outside"):
        crf.dense_crf(img.to(cuda_dev), bad.to(cuda_dev), 2)
    with pytest.raises(_lib.IrnError):
        crf.dense_crf(img.to(cuda_dev), lab.to(cuda_dev), crf.max_labels() + 1)
    rc = _lib.lib().irn_dense_crf(None, None, 1, 8, 8, crf.max_labels() + 1, 10, 0.7, 3, 3, 50, 5, 10, None, None, None, None, 0, None)
    assert rc == -4
    with pytest.raises(_lib.IrnError):
        crf.ir_labels(img.to(cuda_dev), [np.zeros((40, 8, 8), np.float32)], [np.arange(40)], 0.3, 0.05)


@pytest.fixture(scope="module")
def voc_tree(tmp_path_factory, cuda_dev):
    g = np.load(golden_path("steps.npz"))
    root = tmp_path_factory.mktemp("voc_crf")
    os.makedirs(root / "JPEGImages")
    ids = [str(s) for s in g["ids"]]
    labels = {}
    for i, name in enumerate(ids):
        Image.fromarray(g["img%d" % i]).save(root / "JPEGImages" / (name + ".jpg"), format="PNG")
        labels[int(name.replace("_", ""))] = g["label%d" % i]
    (root / "list.txt").write_text("\n".join(ids) + "\n")
    for d in ("sess", "cam", "ir", "ir1"):
        os.makedirs(root / d)
    torch.save(synth.cam_state_dict(), root / "sess" / "res50_cam.pth.pth")
    args = types.SimpleNamespace(
        num_workers=0, voc12_root=str(root), train_list=str(root / "list.txt"), cam_network="irn_b200.cam",
        cam_scales=(1.0, 0.5, 1.5, 2.0), cam_weights_name=str(root / "sess" / "res50_cam.pth"), cam_out_dir=str(root / "cam"),
        ir_label_out_dir=str(root / "ir"), conf_fg_thres=0.30, conf_bg_thres=0.05, synthetic=0)
    from irn_b200.voc12 import dataloader
    dataloader._cls_labels["voc12/cls_labels.npy"] = labels
    return ids, args


def test_step_end_to_end_and_step_batch_identical(voc_tree):
    """make_cam.run then cam_to_ir_label.run: one uint8 PNG per image, the image's size, the reference's name; --step_batch 1
    (the reference's loop) writes the same bytes' pixels as the batched default."""
    ids, args = voc_tree
    from irn_b200.step import cam_to_ir_label, make_cam
    make_cam.run(args)
    cam_to_ir_label.run(args)
    one = types.SimpleNamespace(**vars(args))
    one.step_batch, one.ir_label_out_dir = 1, os.path.join(os.path.dirname(args.ir_label_out_dir), "ir1")
    cam_to_ir_label.run(one)
    g = np.load(golden_path("steps.npz"))
    for i, name in enumerate(ids):
        a = np.asarray(Image.open(os.path.join(args.ir_label_out_dir, name + ".png")))
        b = np.asarray(Image.open(os.path.join(one.ir_label_out_dir, name + ".png")))
        assert a.dtype == np.uint8 and a.shape == g["img%d" % i].shape[:2]
        assert np.array_equal(a, b)
        d = np.load(os.path.join(args.cam_out_dir, name + ".npy"), allow_pickle=True).item()
        ref = ocrf.cam_to_ir_label_one(g["img%d" % i], d["high_res"], d["keys"].numpy())["conf"]
        assert (a != ref).mean() <= 1e-3


def test_multi_gpu_spawn_matches_single(voc_tree):
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the spawn branch is not taken")
    ids, args = voc_tree
    from irn_b200.step import cam_to_ir_label
    cam_to_ir_label.run(args)       # more than one visible GPU: one spawned worker per GPU
    g = np.load(golden_path("steps.npz"))
    for i, name in enumerate(ids):
        a = np.asarray(Image.open(os.path.join(args.ir_label_out_dir, name + ".png")))
        d = np.load(os.path.join(args.cam_out_dir, name + ".npy"), allow_pickle=True).item()
        assert (a != ocrf.cam_to_ir_label_one(g["img%d" % i], d["high_res"], d["keys"].numpy())["conf"]).mean() <= 1e-3


def test_run_sample_writes_ir_labels(tmp_path, cuda_dev):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "run_sample.py"), "--synthetic", "2", "--num_workers", "0",
                        "--make_ins_seg_pass", "False", "--make_sem_seg_pass", "False"], cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "step.cam_to_ir_label is outside" not in r.stdout
    files = sorted(os.listdir(tmp_path / "result" / "ir_label"))
    assert files == ["2007_000000.png", "2007_000001.png"]
    for f in files:
        a = np.asarray(Image.open(tmp_path / "result" / "ir_label" / f))
        assert a.dtype == np.uint8 and a.shape == (512, 512)
