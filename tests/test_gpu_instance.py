"""Instance path kernels: integer outputs bit-exact against the reference's own functions (golden fixtures) and
the oracle."""
import functools

import numpy as np
import pytest
import torch

from conftest import golden_path
from irn_b200 import indexing, instance, pipeline, synth
from oracle import steps
from test_instance_cases_cpu import (CC_PATTERNS, DETECT_CLASSES, DETECT_SIZES, LANDING_CASES, NAN_CHANNEL, cc_pattern,
                                     cc_reference, checker_weak_field, clip_field, detect_case, detect_max_fragment, landing_field, strong_field,
                                     thres_field)

pytestmark = pytest.mark.gpu


def test_find_centroids_bit_exact(cuda_dev):
    g = np.load(golden_path("instance_fns.npz"))
    for i in range(3):
        cen = instance.find_centroids_with_refinement(torch.from_numpy(g["dp%d" % i]).to(cuda_dev))
        assert np.array_equal(cen.cpu().numpy(), g["centroids%d" % i])
    # fewer iterations / noisy field against the oracle
    dp = synth.displacement(37, 61, 4, seed=9) + np.random.default_rng(1).normal(0, 0.5, (2, 37, 61)).astype(np.float32)
    cen = instance.find_centroids_with_refinement(torch.from_numpy(dp).to(cuda_dev), iterations=50)
    assert np.array_equal(cen.cpu().numpy(), steps.find_centroids(dp, 50))


def test_cluster_centroids_exact(cuda_dev):
    g = np.load(golden_path("instance_fns.npz"))
    for i in range(3):
        shape = tuple(g["instances_shape%d" % i])
        ref = np.unpackbits(g["instances%d" % i], axis=-1, count=shape[-1]).astype(bool).reshape(shape)
        inst, n = instance.cluster_centroids(torch.from_numpy(g["centroids%d" % i]).to(cuda_dev), torch.from_numpy(g["dp%d" % i]).to(cuda_dev))
        assert n == shape[0]
        got = steps.one_hot(inst.cpu().numpy(), n)
        assert np.array_equal(got, ref)


def test_connected_components_vs_scipy(cuda_dev):
    rng = np.random.default_rng(3)
    for (h, w, nv) in [(64, 64, 1), (97, 131, 3), (512, 512, 4), (1, 17, 2), (33, 1, 1)]:
        vals = (rng.random((h, w)) < 0.6).astype(np.int32) * rng.integers(1, nv + 1, (h, w)).astype(np.int32)
        lab = instance.connected_components(torch.from_numpy(vals).to(cuda_dev)).cpu().numpy()
        assert ((lab == 0) == (vals == 0)).all()
        for v in range(1, nv + 1):   # per value, same partition as scipy and raster-order numbering
            ref = steps.cc_label(vals == v)
            m = vals == v
            ids = np.unique(lab[m])
            assert len(ids) == ref.max()
            assert np.array_equal(np.searchsorted(ids, lab[m]) + 1, ref[m])


def test_instance_seeds_and_detect(cuda_dev):
    rng = np.random.default_rng(5)
    K, I, h, w = 2, 3, 20, 24
    cams = rng.random((K, h, w)).astype(np.float32)
    inst = rng.integers(0, I, (h, w)).astype(np.int32)
    out = instance.separate_score_by_mask(torch.from_numpy(cams).to(cuda_dev), torch.from_numpy(inst).to(cuda_dev), I).cpu().numpy()
    ref = cams[:, None] * steps.one_hot(inst, I)[None].astype(np.float32)
    assert np.array_equal(out, ref)
    # detect_instance against the oracle restatement
    H, W, C = 60, 72, 4
    idx = (rng.integers(0, C + 1, (H // 6, W // 6)).repeat(6, 0).repeat(6, 1)).astype(np.int32)
    sc = rng.random((C, H, W)).astype(np.float32)
    got = instance.detect_instance(torch.from_numpy(sc).to(cuda_dev), torch.from_numpy(idx).to(cuda_dev), [3, 3, 7, 7], max_fragment_size=40)
    ref = steps.detect_instance(sc, steps.one_hot(idx, C + 1)[1:], [3, 3, 7, 7], max_fragment_size=40)
    assert np.array_equal(got["mask"], ref["mask"]) and np.array_equal(got["class"], ref["class"])
    assert np.array_equal(got["score"].astype(np.float32), np.asarray(ref["score"], np.float32))


# ------------------------------------------------------------------ exact cases at the sizes the steps run (test_instance_cases_cpu.py
# builds them and checks, without a GPU, that each has the property it is meant to have)

STEP_GRIDS = [(94, 125), (125, 94), (128, 128), (160, 160), (160, 107)]      # strided grids of 375x500 ... 640x427 images
ATTRACTORS = [1, 7, 13, 40, 24]


@functools.lru_cache(maxsize=None)
def _step_field(h, w, n_attractors):
    """synth displacement with `n_attractors` attractors, scaled by 3 so that their weak discs (radius ~4) stay apart, plus
    N(0, 0.5) noise; and the oracle's centroids at 300 iterations."""
    dp = 3 * synth.displacement(h, w, n_attractors, seed=n_attractors) + np.random.default_rng(h * w).normal(0, 0.5, (2, h, w))
    dp = dp.astype(np.float32)
    return dp, steps.find_centroids(dp)


def _same_scores(got, ref):
    """Raw float32 bits, except that a NaN must meet a NaN (the device's is 0x7fffffff, x86's 0xffc00000)."""
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    assert got.shape == ref.shape
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got[~nan].view(np.uint32), ref[~nan].view(np.uint32))


def _same_detections(got, ref):
    assert (got is None) == (ref is None)
    if ref is None:
        return
    assert len(got["score"]) == len(ref["score"])
    assert np.array_equal(np.asarray(got["class"]), np.asarray(ref["class"]))
    assert got["mask"].dtype == np.bool_ and np.array_equal(got["mask"], ref["mask"])
    _same_scores(got["score"], ref["score"])


@pytest.mark.parametrize("name", sorted(CC_PATTERNS))
def test_connected_components_exact(cuda_dev, name):
    """Label = 0 on background, else 1 + the smallest flat index of the component: detect_instance reads a segment's channel at
    that pixel.  Spanning components, spirals and combs make the atomicMin links race across blocks along long chains."""
    vals = cc_pattern(name)
    v = torch.from_numpy(np.array(vals)).to(cuda_dev)      # a writable copy of the cached pattern
    a = instance.connected_components(v).cpu().numpy()
    assert np.array_equal(a, cc_reference(vals))
    assert np.array_equal(instance.connected_components(v).cpu().numpy(), a)


def _cluster_exact(cuda_dev, cen, dp, one_hot=True):
    inst, n = instance.cluster_centroids(torch.from_numpy(np.ascontiguousarray(cen)).to(cuda_dev), torch.from_numpy(dp).to(cuda_dev))
    got = inst.cpu().numpy()
    if one_hot:
        ref = steps.cluster_centroids(cen, dp)
        assert n == ref.shape[0]
        assert np.array_equal(steps.one_hot(got, n), ref)
    else:   # too many instances for the one-hot planes: the map they are made from
        ref = steps.cluster_map(cen, dp)
        assert n == ref.max() + 1 and np.array_equal(got, ref)
    return n


@pytest.mark.parametrize("h,w,n_att", [g + (n,) for g, n in zip(STEP_GRIDS, ATTRACTORS)])
def test_cluster_centroids_step_grids(cuda_dev, h, w, n_att):
    dp, cen = _step_field(h, w, n_att)
    assert _cluster_exact(cuda_dev, cen, dp) >= min(n_att, 7)


def test_cluster_centroids_constructed(cuda_dev):
    dp = thres_field()   # strength exactly 2.5 is not weak
    assert _cluster_exact(cuda_dev, steps.find_centroids(dp, 0), dp) == 4
    dp = checker_weak_field()   # 12 801 present values: nearly every thread of rank_scan_kernel carries a partial sum
    assert _cluster_exact(cuda_dev, steps.find_centroids(dp, 0), dp, one_hot=False) == 160 * 160 // 2 + 1
    dp = strong_field()   # no weak pixel
    assert _cluster_exact(cuda_dev, steps.find_centroids(dp, 0), dp) == 1


def _centroids(cuda_dev, dp, its):
    return instance.find_centroids_with_refinement(torch.from_numpy(dp).to(cuda_dev), iterations=its).cpu().numpy()


@pytest.mark.parametrize("h,w,n_att", [g + (n,) for g, n in zip(STEP_GRIDS, ATTRACTORS)])
def test_find_centroids_step_grids(cuda_dev, h, w, n_att):
    dp, cen = _step_field(h, w, n_att)
    assert np.array_equal(_centroids(cuda_dev, dp, 300), cen)
    for its in (0, 1):
        assert np.array_equal(_centroids(cuda_dev, dp, its), steps.find_centroids(dp, its))


def test_find_centroids_clipped_at_both_edges(cuda_dev):
    for h, w, seed in ((61, 47, 0), (160, 107, 1)):
        dp = clip_field(h, w, seed)
        for its in (1, 2, 300):
            assert np.array_equal(_centroids(cuda_dev, dp, its), steps.find_centroids(dp, its)), (h, w, its)


@pytest.mark.parametrize("h,w,its", LANDING_CASES)
def test_find_centroids_exact_landings(cuda_dev, h, w, its):
    """Final positions on exact .5 values (rintf and np.round both round half to even) and on exact integers (uy == ly)."""
    dp = landing_field(h, w, seed=its)
    assert np.array_equal(_centroids(cuda_dev, dp, its), steps.find_centroids(dp, its))


@pytest.mark.parametrize("K,I,h,w", [(80, 3, 94, 125), (80, 200, 23, 37), (3, 300, 41, 67), (20, 57, 107, 160), (1, 1, 5, 7)])
def test_instance_seeds_many(cuda_dev, K, I, h, w):
    rng = np.random.default_rng(K * I)
    cams = rng.random((K, h, w)).astype(np.float32)
    inst = rng.integers(0, I, (h, w)).astype(np.int32)
    out = instance.separate_score_by_mask(torch.from_numpy(cams).to(cuda_dev), torch.from_numpy(inst).to(cuda_dev), I).cpu().numpy()
    assert np.array_equal(out, cams[:, None] * steps.one_hot(inst, I)[None].astype(np.float32))


def _nan_plane(cuda_dev, H, W):
    """The score plane rw_labels gives for an all-zero walk: 0 / 0 everywhere."""
    h, w = (H - 1) // 4 + 1, (W - 1) // 4 + 1
    _, _, sc = indexing.rw_labels(torch.zeros((1, h, w), device=cuda_dev), None, (H, W), want_scores=True)
    return sc[0].cpu().numpy()


@pytest.mark.parametrize("H,W", DETECT_SIZES)
def test_detect_instance_exact(cuda_dev, H, W):
    scores, index = detect_case(H, W, seed=H + W, nan_plane=_nan_plane(cuda_dev, H, W))
    assert np.isnan(scores[NAN_CHANNEL - 1]).all()
    mfs = detect_max_fragment(H, W)
    got = instance.detect_instance(torch.from_numpy(scores).to(cuda_dev), torch.from_numpy(index).to(cuda_dev), DETECT_CLASSES,
                                   max_fragment_size=mfs)
    ref = steps.detect_instance(scores, steps.one_hot(index, len(DETECT_CLASSES) + 1)[1:], DETECT_CLASSES, max_fragment_size=mfs)
    _same_detections(got, ref)


def test_detect_instance_without_segments_raises(cuda_dev):
    scores = np.random.default_rng(0).random((3, 17, 29)).astype(np.float32)
    index = np.zeros((17, 29), np.int32)
    with pytest.raises(ValueError):
        steps.detect_instance(scores, steps.one_hot(index, 4)[1:], [1, 2, 3])
    with pytest.raises(ValueError):
        instance.detect_instance(torch.from_numpy(scores).to(cuda_dev), torch.from_numpy(index).to(cuda_dev), [1, 2, 3])


@pytest.mark.parametrize("C,h,w,H,W", [(20, 94, 125, 375, 497), (64, 57, 61, 227, 243), (150, 40, 27, 159, 107), (300, 40, 50, 157, 198)])
def test_rw_labels_index_mode_many_channels(cuda_dev, C, h, w, H, W):
    """rw_labels as the instance path calls it (keys=None): scores within 1e-6 of the float64 upsample-and-normalise, the index
    equal to the float64 argmax wherever the top-2 margin is above that bound."""
    assert H % 4 and W % 4
    rng = np.random.default_rng(C)
    rw = (rng.random((C, 1, h, w)) ** 3).astype(np.float32)
    rw[:, :, : h // 3] *= 0.2   # the background plane wins somewhere
    _, idx, sc = indexing.rw_labels(torch.from_numpy(rw).to(cuda_dev), None, (H, W), 0.25, want_index=True, want_scores=True)
    up = torch.nn.functional.interpolate(torch.from_numpy(rw).double(), scale_factor=4, mode="bilinear", align_corners=False)
    up = up[:, 0, :H, :W]
    up = (up / up.max()).numpy()     # the max of the cropped planes
    assert np.abs(sc.cpu().numpy() - up).max() < 1e-6
    full = np.concatenate([np.full((1, H, W), 0.25), up], 0)
    got = idx.cpu().numpy()
    bad = got != full.argmax(0)
    assert (got == 0).any() and bad.mean() < 1e-4
    if bad.any():
        srt = np.sort(full, 0)
        assert (srt[-1] - srt[-2])[bad].max() < 1e-6


# ------------------------------------------------------------------ the instance stage end to end, from the walk on

def _stage_inputs(sizes, n_classes, seed):
    """Per image: (keys, strided CAMs fp32 [K,h,w], edge [h,w], displacement [2,h,w]) on its strided grid.  An image whose
    CAMs are all zero walks to zero everywhere: its scores are NaN."""
    rng = np.random.default_rng(seed)
    out = []
    for i, (H, W) in enumerate(sizes):
        h, w = (H - 1) // 4 + 1, (W - 1) // 4 + 1
        K = 1 + i % 3
        keys = np.sort(rng.choice(n_classes, K, replace=False))
        cams = synth.u8_to_cam(synth.cam_planes_u8(K, h, w, seed=seed + i))
        if i == 3:
            cams[:] = 0
        edge = synth.edge_map(h, w, "bimodal", seed=seed + i)[0]
        dp = 2 * synth.displacement(h, w, 3 + 4 * i, seed=seed + i) + rng.normal(0, 0.3, (2, h, w)).astype(np.float32)
        out.append((keys, cams, edge, dp.astype(np.float32)))
    return out


def _oracle_detections(inputs, sizes, walk, dev):
    """The oracle composed stage by stage from the device's walk and rw_labels: centroids, clusters, seeds and detections are
    the oracle's.  `walk(list of seeds [K*I,h,w] cuda)` -> list of walks [K*I,h,w]."""
    seeds, n_inst = [], []
    for keys, cams, edge, dp in inputs:
        inst = steps.cluster_centroids(steps.find_centroids(dp), dp)
        s = cams[:, None] * inst[None].astype(np.float32)
        n_inst.append(s.shape[1])
        seeds.append(s.reshape(-1, *s.shape[2:]))
    rws = walk([torch.from_numpy(np.ascontiguousarray(s)).to(dev) for s in seeds])
    out = []
    for (keys, _, _, _), rw, I, (H, W) in zip(inputs, rws, n_inst, sizes):
        _, index, scores = indexing.rw_labels(rw, None, (H, W), 0.25, want_index=True, want_scores=True)
        C = rw.shape[0]
        try:
            out.append(steps.detect_instance(scores.cpu().numpy(), steps.one_hot(index.cpu().numpy(), C + 1)[1:], np.repeat(keys, I),
                                             max_fragment_size=H * W * 0.01))
        except ValueError:
            out.append(None)
    return out


def test_instance_stage_exact_voc(cuda_dev):
    sizes = [(375, 500)] * 2
    inputs = _stage_inputs(sizes, 20, seed=21)
    pipe = pipeline.PseudoLabelPipeline(None, None, cuda_dev)
    edges = torch.from_numpy(np.stack([e for _, _, e, _ in inputs])).to(cuda_dev)
    dps = torch.from_numpy(np.stack([d for _, _, _, d in inputs])).to(cuda_dev)
    got = pipe.instance_stage([torch.from_numpy(c).to(cuda_dev) for _, c, _, _ in inputs], [k for k, _, _, _ in inputs], edges, dps, sizes[0])

    def walk(seeds):
        rw, counts = pipe.walk_stage(seeds, edges)
        return list(torch.split(rw, counts))
    ref = _oracle_detections(inputs, sizes, walk, cuda_dev)
    assert all(r is not None for r in ref)
    for g, r in zip(got, ref):
        _same_detections(g, r)


def test_instance_ragged_stage_exact_coco(cuda_dev):
    """Mixed MS COCO sizes, 80 classes: instance_ragged_stage on the 160 x 160 canvas equals the composed oracle, and equals
    instance_stage on each image alone, bit for bit.  The canvas inputs are what irn_ragged_stage gives: edges 1.0 and
    displacements 0 outside each image."""
    sizes = [(427, 640), (640, 480), (375, 500), (333, 500)]
    inputs = _stage_inputs(sizes, 80, seed=40)
    fc = 160
    edges = torch.ones((len(sizes), fc, fc), device=cuda_dev)
    dps = torch.zeros((len(sizes), 2, fc, fc), device=cuda_dev)
    for i, (_, _, e, d) in enumerate(inputs):
        edges[i, :e.shape[0], :e.shape[1]] = torch.from_numpy(e)
        dps[i, :, :e.shape[0], :e.shape[1]] = torch.from_numpy(d)
    pipe = pipeline.PseudoLabelPipeline(None, None, cuda_dev)
    cams = [torch.from_numpy(c).to(cuda_dev) for _, c, _, _ in inputs]
    keys = [k for k, _, _, _ in inputs]
    got = pipe.instance_ragged_stage(cams, keys, edges, dps, sizes)
    ref = _oracle_detections(inputs, sizes, lambda seeds: pipe.walk_padded_stage(seeds, edges, sizes), cuda_dev)
    assert all(r is not None for r in ref) and np.isnan(ref[3]["score"]).all()
    for g, r in zip(got, ref):
        _same_detections(g, r)
    for i, (k, c, e, d) in enumerate(inputs):
        alone = pipe.instance_stage([cams[i]], [k], torch.from_numpy(e[None]).to(cuda_dev), torch.from_numpy(d[None]).to(cuda_dev), sizes[i])
        _same_detections(alone[0], got[i])
