"""The background-threshold sweep without a GPU: the oracle's bucket / suffix-sum formulation equals a literal per-threshold loop
(np.pad + argmax + keys + _voc_eval.confusion, step/eval_cam.py:15-18) exactly; the threshold list parsing and normalisation; the
refusals the C ABI makes before anything is launched; the two driver passes."""
import ctypes

import numpy as np
import pytest

from irn_b200.step import _voc_eval
from oracle import threshold_sweep


def literal(scores, keys, gts, thresholds, n_class):
    out = []
    for t in thresholds:
        preds = []
        for s, k in zip(scores, keys):
            cams = np.pad(s, ((1, 0), (0, 0), (0, 0)), mode="constant", constant_values=t)
            kk = np.pad(np.asarray(k) + 1, (1, 0), mode="constant")
            preds.append(kk[np.argmax(cams, axis=0)])
        out.append(_voc_eval.confusion(preds, gts, n_class))
    return np.stack(out)


def case(seed, n_class, shapes, n_keys, T, on_thresholds=True, nan=False):
    rs = np.random.RandomState(seed)
    thr = np.unique(np.round(rs.uniform(0.0, 1.0, T), 2).astype(np.float32))
    while len(thr) < T:     # exactly T distinct float32 values
        thr = np.unique(np.concatenate([thr, rs.uniform(0, 1, T - len(thr)).astype(np.float32)]))
    scores, keys, gts = [], [], []
    for i, ((H, W), K) in enumerate(zip(shapes, n_keys)):
        s = rs.uniform(0, 1, (K, H, W)).astype(np.float32)
        if K and on_thresholds:     # a third of the pixels exactly at a threshold; some foreground ties
            sel = rs.rand(K, H, W) < 0.33
            s[sel] = thr[rs.randint(0, len(thr), sel.sum())]
            tie = rs.rand(H, W) < 0.2
            s[-1][tie] = s[0][tie]
        if K and nan:
            s[rs.randint(0, K)][rs.rand(H, W) < 0.2] = np.nan
        scores.append(s)
        keys.append(np.sort(rs.choice(n_class - 1, K, replace=False)))
        g = rs.randint(0, n_class, (H, W))
        g[rs.rand(H, W) < 0.1] = -1
        gts.append(g)
    return scores, keys, gts, thr


CASES = {
    "voc_T1": dict(seed=1, n_class=21, shapes=[(7, 9), (5, 4)], n_keys=[2, 1], T=1),
    "voc_T91": dict(seed=2, n_class=21, shapes=[(13, 17), (9, 11), (1, 1)], n_keys=[3, 20, 1], T=91),
    "voc_T256": dict(seed=3, n_class=21, shapes=[(16, 16), (3, 30)], n_keys=[4, 2], T=256),
    "coco81_T91": dict(seed=4, n_class=81, shapes=[(20, 24), (11, 8)], n_keys=[80, 5], T=91),
    "nan_planes": dict(seed=5, n_class=21, shapes=[(12, 10), (6, 6)], n_keys=[3, 1], T=40, nan=True),
    "k0": dict(seed=6, n_class=21, shapes=[(8, 8), (5, 7)], n_keys=[0, 2], T=17),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_literal_loop(name):
    scores, keys, gts, thr = case(**CASES[name])
    n = CASES[name]["n_class"]
    got = threshold_sweep.sweep_confusion(scores, keys, gts, thr, n)
    assert got.dtype == np.int64 and got.shape == (len(thr), n, n)
    assert np.array_equal(got, literal(scores, keys, gts, thr, n))


def test_oracle_ties_and_nan_by_hand():
    """m == t is background; equal foreground maxima go to the lowest key index; a NaN channel wins at every threshold."""
    t = np.float32([0.25, 0.5])
    s = np.float32([[[0.25, 0.5, 0.7, np.nan]], [[0.1, 0.5, 0.7, 0.9]]])     # [2,1,4]
    g = np.array([[1, 1, 1, 1]])
    conf = threshold_sweep.sweep_confusion([s], [np.array([0, 4])], [g], t, 6)
    assert np.array_equal(conf, literal([s], [np.array([0, 4])], [g], t, 6))
    # pixel 0: 0.25 == t0 -> background at both; pixel 1: 0.5 tie -> key 1 at t0, background at t1 (0.5 == t1);
    # pixel 2: 0.7 tie -> key 1 at both; pixel 3: NaN in channel 0 -> key 1 at both
    assert conf[0, 1].tolist() == [1, 3, 0, 0, 0, 0]
    assert conf[1, 1].tolist() == [2, 2, 0, 0, 0, 0]


def test_oracle_refuses_labels_outside_classes():
    s = np.ones((1, 2, 2), np.float32)
    with pytest.raises(ValueError):
        threshold_sweep.sweep_confusion([s], [np.array([30])], [np.zeros((2, 2), int)], np.float32([0.5]), 21)


def test_parse_thresholds():
    assert _voc_eval.parse_thresholds("0.1,0.15,0.2") == [0.1, 0.15, 0.2]
    r = _voc_eval.parse_thresholds("0.05:0.95:0.01")
    assert len(r) == 91 and r[0] == 0.05 and r[-1] == 0.95 and r[10] == 0.15
    assert _voc_eval.parse_thresholds("0.2:0.2:0.1") == [0.2]
    assert _voc_eval.parse_thresholds("0:1:0.25") == [0.0, 0.25, 0.5, 0.75, 1.0]
    assert _voc_eval.parse_thresholds([0.3, 0.1]) == [0.3, 0.1]
    for bad in ("", "a,b", "0.1:0.2", "0.5:0.1:0.1", "0:1:0", "0:1:-0.1", "nan", "0.1,,0.2"):
        with pytest.raises(ValueError):
            _voc_eval.parse_thresholds(bad)


def test_sweep_rounds_sorts_and_dedupes(built_lib):
    """ThresholdSweep compares in float32: inputs that round to one float32 give one row; unsorted input is sorted.  Out-of-range
    counts raise IrnError before any device work."""
    from irn_b200 import _lib, indexing
    sw = indexing.ThresholdSweep([0.3, 0.1, 0.1 + 1e-9, 0.2, np.float32(0.2)], 21, "cuda:0")
    assert sw.thresholds.dtype == np.float32 and sw.thresholds.tolist() == np.float32([0.1, 0.2, 0.3]).tolist()
    assert indexing.ThresholdSweep(np.linspace(0, 1, 256), 129, "cuda:0").thresholds.shape == (256,)
    for thr, n in ((np.linspace(0, 1, 257), 21), ([0.5], 130), ([0.5], 0), ([], 21), ([float("nan")], 21)):
        with pytest.raises(_lib.IrnError):
            indexing.ThresholdSweep(thr, n, "cuda:0")


def test_abi_refusals_before_any_launch(built_lib):
    """irn_threshold_sweep_accumulate checks its host tables and sizes before any CUDA call (dummy device pointers, never
    dereferenced): non-ascending or NaN thresholds, T outside 1..256, n_class outside 1..129, sizes that do not match, a key table
    whose background entry is not 0."""
    dummy = ctypes.c_void_p(0x100000)
    keys = np.array([0, 3, 5], np.int32)

    def call(thr, T=None, n_class=21, source=0, C=2, h=8, w=8, H=8, W=8, k=keys):
        thr = np.ascontiguousarray(thr, np.float32)
        return built_lib.irn_threshold_sweep_accumulate(source, dummy, C, h, w, H, W, k.ctypes.data, dummy, thr.ctypes.data,
                                                        len(thr) if T is None else T, n_class, dummy, dummy, None)
    for thr, what in (([0.2, 0.1], b"ascending"), ([0.1, 0.1], b"ascending"), ([0.1, np.nan], b"NaN")):
        assert call(thr) == -1 and what in built_lib.irn_last_error()
    assert call(np.linspace(0, 1, 257)) == -1 and b"257 thresholds" in built_lib.irn_last_error()
    assert call([0.5], T=0) == -1
    assert call([0.5], n_class=130) == -1 and b"n_class=130" in built_lib.irn_last_error()
    assert call([0.5], H=9) == -1 and b"do not match" in built_lib.irn_last_error()
    assert call([0.5], source=1, h=2, w=2, H=9, W=8) == -1 and b"do not match" in built_lib.irn_last_error()
    assert call([0.5], k=np.array([1, 3, 5], np.int32)) == -1 and b"background" in built_lib.irn_last_error()
    assert call([0.5], source=2) == -1 and b"source" in built_lib.irn_last_error()
    assert built_lib.irn_rw_last_launch_count() == 0
    assert built_lib.irn_threshold_sweep_bytes(257, 21) == 0 and built_lib.irn_threshold_sweep_bytes(91, 21) == 21 * 21 * 92 * 8 + 16


def test_driver_flags_and_passes():
    import run_sample
    a = run_sample.parse([])
    assert not a.sweep_cam_pass and not a.sweep_sem_seg_pass
    assert len(a.cam_eval_thres_sweep) == 91 and a.cam_eval_thres_sweep == a.sem_seg_bg_thres_sweep
    assert a.cam_eval_thres == 0.15 and a.sem_seg_bg_thres == 0.25 and a.eval_cam_pass and a.eval_sem_seg_pass
    b = run_sample.parse(["--cam_eval_thres_sweep", "0.1,0.2", "--sem_seg_bg_thres_sweep", "0.2:0.4:0.1", "--sweep_cam_pass", "True"])
    assert b.cam_eval_thres_sweep == (0.1, 0.2) and b.sem_seg_bg_thres_sweep == (0.2, 0.3, 0.4) and b.sweep_cam_pass
    with pytest.raises(SystemExit):
        run_sample.parse(["--cam_eval_thres_sweep", "0.1:x:0.1"])
    P = run_sample.PASSES
    assert P.index("sweep_cam") == P.index("eval_cam") + 1 and P.index("sweep_sem_seg") == P.index("eval_sem_seg") + 1
    assert {"sweep_cam", "sweep_sem_seg"} <= run_sample.PASS_DEFAULT_OFF
    assert run_sample.EVAL_STEPS["sweep_cam"] == "sweep_cam" and run_sample.EVAL_STEPS["sweep_sem_seg"] == "sweep_sem_seg"
