"""The CRF oracle (oracle/crf.py) on the CPU: lattice invariants, the lattice filter against an exact Gaussian filter, CRF
properties that hold exactly, and the cam_to_ir_label step body against tests/golden/ir_label.npz (the unmodified reference's
step with the oracle as its pydensecrf)."""
import hashlib

import numpy as np
import pytest

from conftest import golden_path
from irn_b200 import synth
from oracle import crf


@pytest.mark.parametrize("d", [2, 5])
def test_lattice_invariants(d):
    rs = np.random.RandomState(d)
    f = (rs.rand(2000, d) * 30 - 5).astype(np.float32)
    E, rem0, rank, bary = crf.elevate(f)
    w = bary[:, :d + 1]
    assert w.min() >= 0
    assert np.abs(w.sum(1) - 1).max() < 1e-6
    co = crf.vertex_coords(rem0, rank)                                   # [N, d+1 vertices, d+1 coordinates]
    assert (co.sum(2) == 0).all()                                        # on the hyperplane
    classes = np.sort(co[:, :, 0] % (d + 1), 1)
    assert (classes == np.arange(d + 1)[None]).all()                     # distinct remainder classes
    assert all((co[:, r] % (d + 1) == r).all() for r in range(d + 1))
    rec = (w[:, :, None].astype(np.float64) * co).sum(1)
    assert np.abs(rec - E).max() < 1e-4                                  # the weights reproduce the elevated point


@pytest.mark.parametrize("d,H,W,bound,sigma_band", [(2, 40, 40, 0.995, (0.9, 1.2)), (5, 30, 30, 0.93, (0.7, 1.1))])
def test_lattice_filter_approximates_gaussian(d, H, W, bound, sigma_band):
    """L(v) against the exact filter sum_j exp(-|f_i - f_j|^2 / (2 s^2)) v_j over a grid of widths s.  Measured here: d=2
    correlation 0.9988 at s = 1.05, d=5 correlation 0.946 at s = 0.85 (random features in [0, 8)^d)."""
    rs = np.random.RandomState(0)
    f = (rs.rand(H * W, d) * 8).astype(np.float32)
    v = rs.rand(H * W, 1).astype(np.float32)
    out = crf.Lattice(f).compute(v)[:, 0].astype(np.float64)
    D2 = ((f[:, None, :].astype(np.float64) - f[None, :, :]) ** 2).sum(-1)
    best = max((np.corrcoef(out, np.exp(-D2 / (2 * s * s)) @ v[:, 0])[0, 1], s) for s in np.arange(0.5, 3.0, 0.05))
    assert best[0] > bound, best
    assert sigma_band[0] <= best[1] <= sigma_band[1], best


def test_unary_from_labels():
    lab = np.array([[0, 2], [1, 2]])
    U = crf.unary_from_labels(lab, 3, gt_prob=0.7)
    assert U.dtype == np.float32 and U.shape == (3, 4)
    pe, ne = np.float32(-np.log(0.7)), np.float32(-np.log(0.3 / 2))
    want = np.full((3, 4), ne, np.float32)
    want[lab.reshape(-1), np.arange(4)] = pe
    assert np.array_equal(U, want)
    U1 = crf.unary_from_labels(np.zeros((2, 3), int), 1, gt_prob=0.7)     # no other label: no divisor
    assert np.array_equal(U1, np.full((1, 6), pe, np.float32))
    with pytest.raises(ValueError):
        crf.unary_from_labels(lab, 2, gt_prob=0.7)


def test_single_label_is_all_zero():
    img = synth.image(3, 20, 24)
    assert (crf.crf_inference_label(img, np.zeros((20, 24), int), n_labels=1) == 0).all()
    q = crf.crf_inference_q(img, np.zeros((20, 24), int), n_labels=1)
    assert (q == 1).all()


def test_compat_zero_returns_input_labels():
    rs = np.random.RandomState(1)
    img = synth.image(4, 30, 40)
    lab = rs.randint(0, 4, (30, 40))
    q = crf.crf_inference_q(img, lab, t=5, n_labels=4, gauss=(3, 0), bilateral=(50, 5, 0))
    assert np.array_equal(np.argmax(q, 0), lab)


def test_salt_noise_removed_boundaries_kept():
    H, W = 48, 64
    regions = np.zeros((H, W), int)
    regions[:, 32:] = 1
    regions[24:, :20] = 2
    colours = np.array([[200, 30, 30], [30, 200, 30], [30, 30, 200]], np.uint8)
    img = colours[regions]
    rs = np.random.RandomState(2)
    noisy = regions.copy()
    salt = rs.rand(H, W) < 0.08
    noisy[salt] = rs.randint(0, 3, salt.sum())
    assert (noisy != regions).sum() > 50
    out = crf.crf_inference_label(img, noisy, n_labels=3)
    assert np.array_equal(out, regions)


def _fixture_case(g, i):
    if ("seed%d" % i) in g:
        H, W = g["png%d" % i].shape
        keys = g["keys%d" % i]
        u8 = synth.cam_planes_u8(len(keys), H, W, int(g["seed%d" % i]))
        assert hashlib.sha256(np.ascontiguousarray(u8).tobytes()).hexdigest() == str(g["cam_sha256%d" % i]), \
            "synth.cam_planes_u8 no longer regenerates the fixture's CAM planes"
        return synth.image(int(g["seed%d" % i]), H, W), synth.u8_to_cam(u8)
    j = int(g["steps_index%d" % i])
    return STEPS["img%d" % j], STEPS["cam_high%d" % j].astype(np.float32)


G = np.load(golden_path("ir_label.npz"))
STEPS = np.load(golden_path("steps.npz"))


@pytest.mark.parametrize("i", range(int(G["n"])))
def test_oracle_step_reproduces_reference_step(i):
    img, high = _fixture_case(G, i)
    got = crf.cam_to_ir_label_one(img, high, G["keys%d" % i], float(G["conf_fg_thres"]), float(G["conf_bg_thres"]),
                                    with_q=("q_fg%d" % i) in G)
    for k in ("fg_conf_cam", "bg_conf_cam", "pred_fg", "pred_bg"):
        assert np.array_equal(got[k], G[k + "%d" % i]), k
    assert np.array_equal(got["conf"], G["png%d" % i])
    if ("q_fg%d" % i) in G:
        assert np.array_equal(got["q_fg"], G["q_fg%d" % i])
