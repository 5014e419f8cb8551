"""Every device entry point honours the caller's stream (include/irn_b200.h: all work is enqueued on the caller's stream, in order).

Late inputs.  On a side stream (PyTorch makes it non-blocking: it does not wait for the legacy default stream) the inputs are
allocated, filled with poison, held back by one bounded `torch.cuda._sleep` of about 20 ms and only then overwritten with the real
data; the entry point is called under `torch.cuda.stream(side)` right away, and the test waits for that stream alone.  A launch,
memset, CUB pass or copy of the call that ran on any other stream would have run during the sleep and read the poison, so the result
must equal, bit for bit, the same call on the default stream with ready inputs; where a cheap oracle exists the case is also held to
it.  The poison is NaN for float inputs and a valid but wrong value (zeros) for index-like ones (labels, maps, centroids), so a
wrong-stream bug shows as wrong values, never as an out-of-range access.

Consumption on another stream: the default stream waits for the side stream (`wait_stream`) and reads the outputs with no other
synchronisation; host values the wrappers return (instance count, detections, CRF vertex counts) are the synchronised ones.

Shared caches: the workspace and scratch buffers the wrappers keep (indexing._workspace / _scratch, cam_ops' and preprocess'
buffers) belong to one (device, stream), so two streams never share bytes and growing one stream's buffer never hands a block that
another stream's queued call uses back to the allocator.  Two host threads on two streams, one walking at radius 5 and the other at
radius 3 and 10, get the serial results, and the per-thread state of the library stays per thread.

Every case runs once; nothing loops to catch a race."""
import ctypes
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from conftest import golden_path
from irn_b200 import _lib, cam_ops, crf, indexing, instance, preprocess, synth
from oracle import crf as ocrf
from oracle import indexing as oi
from oracle import resize as R
from oracle import steps

pytestmark = pytest.mark.gpu

SLEEP_S = 0.02
SM_CLOCK_HZ = 1.98e9                      # the H100 SXM's highest SM clock: at any lower clock the sleep lasts longer
SLEEP_CYCLES = int(SLEEP_S * SM_CLOCK_HZ)
NAN = float("nan")


# ------------------------------------------------------------------------------------------------------------------- harness
@pytest.fixture(scope="module")
def side(cuda_dev):
    return torch.cuda.Stream(cuda_dev)


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _host(v):
    """Tensors -> numpy (read on the current stream), recursively through tuples, lists and dicts."""
    if isinstance(v, torch.Tensor):
        return v.detach().cpu().numpy()
    if isinstance(v, (list, tuple)):
        return type(v)(_host(x) for x in v)
    if isinstance(v, dict):
        return {k: _host(x) for k, x in v.items()}
    return v


def assert_same(got, want, what="result"):
    """Bit for bit, through containers; numpy scalars and Python values by equality."""
    if isinstance(want, np.ndarray):
        got = np.asarray(got)
        assert got.shape == want.shape and got.dtype == want.dtype, "%s: %s %s != %s %s" % (what, got.shape, got.dtype, want.shape, want.dtype)
        assert got.tobytes() == want.tobytes(), "%s: %d of %d elements differ" % (
            what, int((got.reshape(-1).view(np.uint8) != want.reshape(-1).view(np.uint8)).sum()), want.size)
    elif isinstance(want, (list, tuple)):
        assert len(got) == len(want), what
        for i, (g, w) in enumerate(zip(got, want)):
            assert_same(g, w, "%s[%d]" % (what, i))
    elif isinstance(want, dict):
        assert sorted(got) == sorted(want), what
        for k in want:
            assert_same(got[k], want[k], "%s[%r]" % (what, k))
    else:
        assert got == want, "%s: %r != %r" % (what, got, want)


def late(stream, srcs, poisons):
    """Copies of the ready device tensors `srcs` that hold `poisons` (a fill value or a tensor of the same shape) on `stream` until
    a sleep of SLEEP_CYCLES has passed there.  The sources are recorded on `stream`, so that the caller may drop them at once: their
    blocks go back to the allocator only after the delayed copies."""
    stream.wait_stream(torch.cuda.default_stream(stream.device))          # the sources and poisons exist
    for t in list(srcs) + [p for p in poisons if isinstance(p, torch.Tensor)]:
        t.record_stream(stream)
    with torch.cuda.stream(stream):
        bufs = [torch.empty_like(s) for s in srcs]
        for b, p in zip(bufs, poisons):
            if isinstance(p, torch.Tensor):
                b.copy_(p)
            else:
                b.fill_(p)
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, s in zip(bufs, srcs):
            b.copy_(s)
    return bufs


def on_side(side, fn, srcs, poisons, consume_on_default=False, late_first=False):
    """fn(*srcs) on the default stream with ready inputs, and fn on late inputs on `side` (after it with late_first): returns
    (ready, late) results as host data.  consume_on_default: instead of waiting for `side`, the default stream waits for it and
    reads the results."""
    want = None if late_first else _host(fn(*srcs))
    ins = late(side, srcs, poisons)
    with torch.cuda.stream(side):
        got = fn(*ins)
    if consume_on_default:
        torch.cuda.default_stream(side.device).wait_stream(side)
    else:
        side.synchronize()
    got = _host(got)
    return (_host(fn(*srcs)) if late_first else want), got


# ------------------------------------------------------------------------------------------------------- walk and affinities
@pytest.mark.parametrize("h,w", [(16, 24), (13, 29)])
def test_edge_to_affinity_late_edge(cuda_dev, side, h, w):
    e = synth.edge_map(h, w, "uniform", h)
    want, got = on_side(side, lambda x: indexing.edge_to_affinity(x, 5), [_t(e, cuda_dev)], [NAN])
    assert_same(got, want)
    W, _ = oi.stencil_weights(e, 5, beta=1)
    assert np.array_equal(got[0], W)


@pytest.mark.parametrize("h,w,r", [(20, 28, 5), (17, 31, 10)])
def test_to_affinity_forward_backward_late_inputs(cuda_dev, side, h, w, r):
    edge = synth.edge_map(h, w, "bimodal", r).repeat(2, 0) * np.float32(0.9)
    edge[1] = synth.edge_map(h, w, "uniform", r + 1)[0]

    def fwd(x):
        return indexing.to_affinity(x.requires_grad_(True), radius=r)

    e_ref, e_late = _t(edge, cuda_dev), late(side, [_t(edge, cuda_dev)], [NAN])[0]
    a_ref = fwd(e_ref)
    with torch.cuda.stream(side):
        a_late = fwd(e_late)
    side.synchronize()
    aff, arg = oi.to_affinity(edge, oi.PathIndex(r, (h, w)).path_indices)
    assert_same(_host(a_late), _host(a_ref), "aff")
    assert np.array_equal(_host(a_late), aff)
    # backward: autograd runs it on the forward's stream; the incoming gradient is late there too.  The scatter adds with atomics,
    # so the gradient is held to the fp64 oracle at the tolerance of test_gpu_random_walk, not bit for bit.
    g = np.random.default_rng(r).standard_normal(tuple(a_ref.shape)).astype(np.float32)
    g_late = late(side, [_t(g, cuda_dev)], [NAN])[0]
    with torch.cuda.stream(side):
        a_late.backward(g_late)
    side.synchronize()
    truth = oi.to_affinity_backward(g, arg, h * w).reshape(2, h, w)
    assert np.abs(_host(e_late.grad) - truth).max() < 1e-5 * max(1.0, float(np.abs(truth).max()))


@pytest.mark.parametrize("variant", [0, 1, 2, 4])
@pytest.mark.parametrize("h,w", [(40, 36), (33, 47)])
def test_random_walk_late_inputs(cuda_dev, side, variant, h, w):
    C = 3
    x, e = synth.seeds(C, h, w, h), synth.edge_map(h, w, "bimodal", w)
    walk = lambda xs, es: indexing.random_walk_batch(xs, es, [0, C], 5, 10, 16, variant=variant)
    want, got = on_side(side, walk, [_t(x, cuda_dev), _t(e, cuda_dev)], [NAN, NAN])
    assert_same(got, want)
    assert np.abs(got - oi.propagate_stencil(x, e, 5, 10, 16).reshape(C, h, w)).max() < 1e-6


def test_random_walk_mixed_channels_consumed_on_default(cuda_dev, side):
    h, w = 40, 36
    counts = [2, 0, 1, 6, 3]
    offs = np.concatenate([[0], np.cumsum(counts)])
    edges = np.concatenate([synth.edge_map(h, w, "bimodal", i) for i in range(len(counts))], 0)
    x = synth.seeds(int(offs[-1]), h, w, 99)
    walk = lambda xs, es: indexing.random_walk_batch(xs, es, offs, n_iter=32)
    want, got = on_side(side, walk, [_t(x, cuda_dev), _t(edges, cuda_dev)], [NAN, NAN], consume_on_default=True)
    assert_same(got, want)
    for i, c in enumerate(counts):
        if c:
            truth = oi.propagate_stencil(x[offs[i]:offs[i + 1]], edges[i], 5, 10, 32).reshape(c, h, w)
            assert np.abs(got[offs[i]:offs[i + 1]] - truth).max() < 1e-6


def test_radius_switch_inside_a_late_walk(cuda_dev, side):
    """A walk at radius 3, then one at radius 5, both on late inputs and before their default-stream twins: each late call uploads
    its radius' tables."""
    h, w, C = 30, 33, 2
    x, e = synth.seeds(C, h, w, 5), synth.edge_map(h, w, "uniform", 5)
    for r in (3, 5):
        walk = lambda xs, es: indexing.random_walk_batch(xs, es, [0, C], radius=r, n_iter=8)
        want, got = on_side(side, walk, [_t(x, cuda_dev), _t(e, cuda_dev)], [NAN, NAN], late_first=True)
        assert_same(got, want, "radius %d" % r)
        assert np.abs(got - oi.propagate_stencil(x, e, r, 10, 8).reshape(C, h, w)).max() < 1e-6


@pytest.mark.parametrize("C,h,w,H,W", [(2, 24, 32, 96, 128), (3, 19, 25, 75, 99)])
def test_rw_labels_late_walk(cuda_dev, side, C, h, w, H, W):
    rng = np.random.default_rng(C)
    rw = rng.random((C, 1, h, w)).astype(np.float32)
    rw[:, :, : h // 2] *= 0.2
    keys = sorted(rng.choice(20, C, replace=False).tolist())
    with_keys = lambda r: indexing.rw_labels(r, keys, (H, W), 0.25)[0]
    want, got = on_side(side, with_keys, [_t(rw, cuda_dev)], [NAN])
    assert_same(got, want, "labels")
    full = lambda r: indexing.rw_labels(r, None, (H, W), 0.25, want_index=True, want_scores=True)
    want, got = on_side(side, full, [_t(rw, cuda_dev)], [NAN], consume_on_default=True)
    assert_same(got, want, "labels, index, scores")
    assert np.abs(got[2] - steps.upsample4_norm(torch.from_numpy(rw), (H, W)).numpy()).max() < 1e-6


def test_merge_cams_late_outputs(cuda_dev, side):
    rs = np.random.RandomState(4)
    H, W = 75, 101
    outs = [rs.rand(20, hs, ws).astype(np.float32) for hs, ws in ((5, 7), (3, 4), (8, 10), (10, 13))]
    label = np.zeros(20, np.float32)
    label[[2, 9, 17]] = 1
    merge = lambda *o: cam_ops.merge_cams(list(o), (H, W), torch.from_numpy(label))
    want, got = on_side(side, merge, [_t(o, cuda_dev) for o in outs], [NAN] * 4)
    assert_same(got, want)
    rk, rlo, rhi = steps.cam_merge([torch.from_numpy(o) for o in outs], (H, W), torch.from_numpy(label))
    assert np.array_equal(got[0], rk.numpy())
    assert np.abs(got[1] - rlo.numpy()).max() < 1e-5 and np.abs(got[2] - rhi.numpy()).max() < 1e-5


# ------------------------------------------------------------------------------------------------------------------ instances
@pytest.mark.parametrize("h,w", [(32, 48), (37, 61)])
def test_instance_path_late_inputs(cuda_dev, side, h, w):
    dp = synth.displacement(h, w, 4, seed=h)
    cen_want, cen = on_side(side, lambda d: instance.find_centroids_with_refinement(d, 50), [_t(dp, cuda_dev)], [NAN])
    assert_same(cen, cen_want, "centroids")
    assert np.array_equal(cen, steps.find_centroids(dp, 50))
    # the centroids are index-like: poisoned with zeros, a valid but wrong field
    cl = lambda c, d: instance.cluster_centroids(c, d)
    want, got = on_side(side, cl, [_t(cen, cuda_dev), _t(dp, cuda_dev)], [0, NAN])
    assert_same(got, want, "cluster_centroids")
    inst_map, n_inst = got
    assert n_inst >= 1 and n_inst == int(inst_map.max()) + 1
    assert np.array_equal(steps.one_hot(inst_map, n_inst), steps.cluster_centroids(cen, dp))
    rng = np.random.default_rng(h)
    cams = rng.random((2, h, w)).astype(np.float32)
    sep = lambda c, m: instance.separate_score_by_mask(c, m, n_inst)
    want, got = on_side(side, sep, [_t(cams, cuda_dev), _t(inst_map, cuda_dev)], [NAN, 0], consume_on_default=True)
    assert_same(got, want, "separate_score_by_mask")
    assert np.array_equal(got, cams[:, None] * steps.one_hot(inst_map, n_inst)[None].astype(np.float32))
    vals = ((rng.random((h, w)) < 0.6) * rng.integers(1, 4, (h, w))).astype(np.int32)
    want, got = on_side(side, instance.connected_components, [_t(vals, cuda_dev)], [0])
    assert_same(got, want, "connected_components")
    for v in range(1, 4):
        m = vals == v
        ids = np.unique(got[m])
        assert np.array_equal(np.searchsorted(ids, got[m]) + 1, steps.cc_label(m)[m])


def test_detect_instance_late_inputs(cuda_dev, side):
    rng = np.random.default_rng(5)
    H, W, C = 60, 78, 4
    idx = (rng.integers(0, C + 1, (H // 6, W // 6)).repeat(6, 0).repeat(6, 1)).astype(np.int32)
    sc = rng.random((C, H, W)).astype(np.float32)
    det = lambda s, i: instance.detect_instance(s, i, [3, 3, 7, 7], max_fragment_size=40)
    want, got = on_side(side, det, [_t(sc, cuda_dev), _t(idx, cuda_dev)], [NAN, 0])
    assert_same(got, want, "detections")
    ref = steps.detect_instance(sc, steps.one_hot(idx, C + 1)[1:], [3, 3, 7, 7], max_fragment_size=40)
    assert np.array_equal(got["mask"], ref["mask"]) and np.array_equal(got["class"], ref["class"])
    assert np.array_equal(got["score"].astype(np.float32), np.asarray(ref["score"], np.float32))


# --------------------------------------------------------------------------------------------------------------- convolutions
def test_conv_modes_stem_and_shortcut_late_inputs(cuda_dev, side):
    """One integer-valued case of each kind from test_conv_exact: exact against fp64, in every mode, on late inputs."""
    from test_conv_exact import (N_SM_STANDIN, SHORTCUT_CASES, STEM_CASES, _conv_cases, _shortcut_reference_inputs, conv_data,
                                 shortcut_data, stem_data)
    from irn_b200.ops import Conv2d, ShortcutConv, Stem
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
    c = next(k for k in _conv_cases(N_SM_STANDIN) if k.id == "odd_37x51_stride2_3x3_ragged")
    x, w, bn, res = conv_data(c)
    ref = F.conv2d(_t(x, cuda_dev).double(), _t(w, cuda_dev).double(), stride=c.stride, padding=c.pad)
    ref = nhwc(ref + _t(bn[1], cuda_dev).double()[:, None, None] + _t(res, cuda_dev).double()).float().cpu().numpy()
    conv = Conv2d(w, bn, c.stride, c.pad)
    for mode in (0, 1, 2):
        f = lambda xs, rs: conv(xs, rs, relu=c.relu, mode=mode)
        want, got = on_side(side, f, [nhwc(_t(x, cuda_dev)), nhwc(_t(res, cuda_dev))], [NAN, NAN])
        assert_same(got, want, "conv mode %d" % mode)
        assert_same(got, ref, "conv mode %d against fp64" % mode)
    s = next(k for k in STEM_CASES if k.id == "30x41_padded_to_48x48")
    x, w, bn = stem_data(s)
    xp = F.pad(_t(x, cuda_dev).double(), (0, s.Win - s.W, 0, s.Hin - s.H))
    ref = nhwc(F.relu(F.conv2d(xp, _t(w, cuda_dev).double(), stride=2, padding=3) + _t(bn[1], cuda_dev).double()[:, None, None]))
    ref = ref.float().cpu().numpy()
    stem = Stem(w, bn)
    for mode in (0, 1, 2):
        want, got = on_side(side, lambda xs: stem(xs, s.Hin, s.Win, mode=mode), [_t(x, cuda_dev)], [NAN])
        assert_same(got, want, "stem mode %d" % mode)
        assert_same(got, ref, "stem mode %d against fp64" % mode)
    k = next(k for k in SHORTCUT_CASES if k.id == "layer2_128_256_s2_2x3_tiles")
    t2, x, w3, wds, bn3, bnds = shortcut_data(k)
    a, wc = _shortcut_reference_inputs(k, t2, x, w3, wds)
    ref = F.conv2d(_t(a, cuda_dev).double(), _t(wc, cuda_dev).double()) + _t(bn3[1] + bnds[1], cuda_dev).double()[:, None, None]
    ref = nhwc(F.relu(ref)).float().cpu().numpy()
    sc = ShortcutConv(w3, bn3, wds, bnds, k.stride)
    want, got = on_side(side, sc, [nhwc(_t(t2, cuda_dev)), nhwc(_t(x, cuda_dev))], [NAN, NAN])
    assert_same(got, want, "shortcut")
    assert_same(got, ref, "shortcut against fp64")


# ------------------------------------------------------------------------------------------------------------------- networks
@pytest.fixture(scope="module")
def cam_model(cuda_dev):
    from irn_b200.cam import CAM
    m = CAM()
    m.load_state_dict(synth.cam_state_dict(), strict=True)
    return m


@pytest.fixture(scope="module")
def irn_model(cuda_dev):
    from irn_b200.irn import EdgeDisplacement
    m = EdgeDisplacement(crop_size=128)
    m.load_state_dict(synth.irn_state_dict(), strict=False)
    return m


def _pair(img):
    x = synth.normalize_image(img)
    return np.stack([x, x[..., ::-1].copy()])


def test_cam_forward_and_ragged_late_inputs(cuda_dev, side, cam_model):
    from oracle import nets
    xi = _pair(synth.image(5, 61, 97))
    want, got = on_side(side, cam_model, [_t(xi, cuda_dev)], [NAN])
    assert_same(got, want, "CAM.forward")
    with torch.no_grad():
        ref = nets.cam_forward(torch.from_numpy(xi), synth.cam_state_dict()).numpy()
    assert np.abs(got - ref).max() / ref.max() < 1e-4
    imgs = [synth.image(7, 37, 51), synth.image(8, 64, 45)]
    canvas, ext = preprocess.resize_normalize_ragged(torch.cat([_t(i, cuda_dev).reshape(-1) for i in imgs]), [i.shape[:2] for i in imgs], 1.0)
    want, got = on_side(side, lambda c: cam_model.forward_ragged(c, ext), [canvas], [NAN], consume_on_default=True)
    assert_same(got, want, "CAM.forward_ragged")
    for i, img in enumerate(imgs):
        one = _host(cam_model.forward_batch(preprocess.msf_batch(_t(img[None], cuda_dev), (1.0,))[0])[0])
        h, w = one.shape[-2:]
        assert_same(got[i][:, :h, :w], one, "corner %d" % i)


def test_edge_displacement_forward_and_ragged_late_inputs(cuda_dev, side, irn_model):
    xi = _pair(synth.image(3, 64, 96))
    want, got = on_side(side, irn_model, [_t(xi, cuda_dev)], [NAN])
    assert_same(got, want, "EdgeDisplacement.forward")
    sizes = [(61, 97), (40, 33), (128, 1)]
    imgs = [synth.image(10 + i, h, w) for i, (h, w) in enumerate(sizes)]
    flat = _t(np.concatenate([i.reshape(-1) for i in imgs]), cuda_dev)
    want, got = on_side(side, lambda f: irn_model.forward_ragged(f, sizes), [flat], [0])
    assert_same(got, want, "EdgeDisplacement.forward_ragged")
    for i, img in enumerate(imgs):
        e, d = _host(irn_model.forward_batch(preprocess.msf_batch(_t(img[None], cuda_dev), (1.0,))[0]))
        fh, fw = e.shape[-2:]
        assert_same(got[0][i, :, :fh, :fw], e[0], "edge %d" % i)
        assert_same(got[1][i, :, :fh, :fw], d[0], "dp %d" % i)


# ---------------------------------------------------------------------------------------------------------------- preprocessing
def _pillow(img, oh, ow):
    return np.asarray(Image.fromarray(img).resize((ow, oh), Image.BICUBIC)) if (oh, ow) != img.shape[:2] else img


def test_resize_normalize_late_images(cuda_dev, side):
    H, W, oh, ow = 37, 50, 56, 75
    imgs = np.stack([synth.image(2, H, W), synth.image(9, H, W)])
    f = lambda x: preprocess.resize_normalize(x, (oh, ow), want_u8=True)
    want, got = on_side(side, f, [_t(imgs, cuda_dev)], [0])
    assert_same(got, want)
    lut = R.normalize_lut()
    for b in range(2):
        ref = _pillow(imgs[b], oh, ow)
        assert np.array_equal(got[1][b], ref)
        assert np.array_equal(got[0][2 * b], np.stack([lut[c][ref[..., c]] for c in range(3)]))
    scales = (1.0, 0.5, 1.5)
    want, got = on_side(side, lambda x: preprocess.msf_batch(x, scales), [_t(imgs[:1], cuda_dev)], [0], consume_on_default=True)
    assert_same(got, want, "msf_batch")
    for g, r in zip(got, R.msf_preprocess(imgs[0], scales)):
        assert np.array_equal(g, r)


def test_resize_normalize_ragged_late_images(cuda_dev, side):
    sizes = [(37, 51), (20, 33), (1, 7)]
    imgs = [synth.image(20 + i, h, w) for i, (h, w) in enumerate(sizes)]
    flat = _t(np.concatenate([i.reshape(-1) for i in imgs]), cuda_dev)
    want, got = on_side(side, lambda f: preprocess.resize_normalize_ragged(f, sizes, 1.5)[0], [flat], [0])
    assert_same(got, want)
    lut = R.normalize_lut()
    for i, img in enumerate(imgs):
        oh, ow = preprocess.rescaled_size(*img.shape[:2], 1.5)
        ref = np.stack([lut[c][_pillow(img, oh, ow)[..., c]] for c in range(3)])
        assert np.array_equal(got[2 * i][:, :oh, :ow], ref) and np.array_equal(got[2 * i + 1][:, :oh, :ow], ref[..., ::-1])


# ------------------------------------------------------------------------------------------------------------------------ JPEG
def test_exact_jpeg_decode_behind_a_busy_stream(cuda_dev, side):
    """Two decodes queued behind a sleep: the first one's pinned staging must stay untouched (the decoder keeps it until an event
    has passed) while the second call stages its own bytes; both equal the fixture's pixels."""
    from irn_b200.jpeg import ExactJpegDecoder
    g = np.load(golden_path("jpeg_exact.npz"))
    cases = [(g["jpeg%d" % i].tobytes(), g["pixels%d" % i]) for i in range(min(6, int(g["n"])))]
    a, b = cases[: len(cases) // 2], cases[len(cases) // 2:]
    dec = ExactJpegDecoder(cuda_dev)
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        fa, sa, st_a = dec.decode_packed([d for d, _ in a], check=False)
        fb, sb, st_b = dec.decode_packed([d for d, _ in b], check=False)
    side.synchronize()
    st_a.check()
    st_b.check()
    for flat, sizes, part in ((fa, sa, a), (fb, sb, b)):
        host, o = flat.cpu().numpy(), 0
        for (h, w), (_, pixels) in zip(sizes, part):
            assert np.array_equal(host[o:o + 3 * h * w].reshape(h, w, 3), pixels)
            o += 3 * h * w


# ------------------------------------------------------------------------------------------------------------------------- CRF
def test_dense_crf_late_inputs_vs_oracle(cuda_dev, side):
    H, W, n = 20, 24, 5
    img = synth.image(3, H, W)
    lab = synth.cam_planes_u8(n, H, W, 3).argmax(0).astype(np.int32)
    f = lambda i, l: crf.dense_crf(i, l, n, t=10, want_q=True)
    want, got = on_side(side, f, [_t(img[None], cuda_dev), _t(lab[None], cuda_dev)], [0, 0])
    assert_same(got, want)
    d = ocrf.DenseCRF2D(W, H, n)
    d.setUnaryEnergy(ocrf.unary_from_labels(lab, n, 0.7))
    d.addPairwiseGaussian(sxy=3, compat=3)
    d.addPairwiseBilateral(sxy=50, srgb=5, rgbim=img, compat=10)
    q_ref = d.inference(10).reshape(n, H, W)
    assert got[2][0].tolist() == [p.lattice.n_vertices for p in d.pairwise]
    assert np.abs(got[1][0] - q_ref).max() < 1e-5


def test_dense_crf_ragged_late_inputs(cuda_dev, side):
    sizes = [(17, 23), (1, 9), (31, 12)]
    imgs = [synth.image(30 + i, h, w) for i, (h, w) in enumerate(sizes)]
    n = 4
    labs = [synth.cam_planes_u8(n, h, w, i).argmax(0).astype(np.int32) for i, (h, w) in enumerate(sizes)]
    flat = _t(np.concatenate([i.reshape(-1) for i in imgs]), cuda_dev)
    lab = _t(np.concatenate([l.reshape(-1) for l in labs]), cuda_dev)
    f = lambda i, l: crf.dense_crf_ragged(i, sizes, l, n, want_q=True)
    want, got = on_side(side, f, [flat, lab], [0, 0], consume_on_default=True)
    assert_same(got, want)
    for i, (h, w) in enumerate(sizes):
        one = crf.dense_crf(_t(imgs[i][None], cuda_dev), _t(labs[i][None], cuda_dev), n, want_q=True)
        assert_same(crf.unpack(torch.from_numpy(got[1]), sizes, n)[i].numpy(), _host(one[1][0]), "Q %d" % i)
        assert got[2][i].tolist() == one[2][0].tolist()


def _conf_case(sizes, seed):
    imgs = [synth.image(seed + i, h, w) for i, (h, w) in enumerate(sizes)]
    keys = [np.sort(np.random.default_rng(seed + i).choice(20, 1 + i % 3, replace=False)) for i in range(len(sizes))]
    high = [synth.u8_to_cam(synth.cam_planes_u8(len(k), h, w, seed + i)) for i, (k, (h, w)) in enumerate(zip(keys, sizes))]
    return imgs, keys, high


def test_ir_labels_late_inputs(cuda_dev, side):
    H, W = 29, 40
    imgs, keys, high = _conf_case([(H, W)] * 2, 40)
    f = lambda i, h0, h1: crf.ir_labels(i, [h0, h1], keys, 0.30, 0.05, return_counts=True)
    want, got = on_side(side, f, [_t(np.stack(imgs), cuda_dev), _t(high[0], cuda_dev), _t(high[1], cuda_dev)], [0, NAN, NAN])
    assert_same(got, want)
    for i in range(2):
        ref = ocrf.cam_to_ir_label_one(imgs[i], high[i], keys[i], 0.30, 0.05)["conf"]
        assert (got[0][i] != ref).mean() <= 1e-3


def test_ir_labels_ragged_late_inputs(cuda_dev, side):
    sizes = [(29, 40), (13, 7), (40, 29)]
    imgs, keys, high = _conf_case(sizes, 50)
    flat = _t(np.concatenate([i.reshape(-1) for i in imgs]), cuda_dev)
    f = lambda i, *h: crf.ir_labels_ragged(i, sizes, list(h), keys, 0.30, 0.05, return_counts=True)
    want, got = on_side(side, f, [flat] + [_t(h, cuda_dev) for h in high], [0] + [NAN] * 3)
    assert_same(got, want)
    for i, (lab, (h, w)) in enumerate(zip(crf.unpack(torch.from_numpy(got[0]), sizes), sizes)):
        one = crf.ir_labels(_t(imgs[i][None], cuda_dev), [high[i]], [keys[i]], 0.30, 0.05)
        assert_same(lab.numpy(), _host(one[0]), "image %d" % i)


# ----------------------------------------------------------------------------------------------------------------- COCO masks
def test_coco_masks_late_inputs(cuda_dev, side):
    from irn_b200.coco import mask as cmask
    from oracle import coco_mask as ocm
    anns = [(10, 12, [[2, 3, 6, 3, 6, 8, 2, 8]], 1), (33, 17, [[1.5, 1, 15, 2.5, 9, 30, -1, 20]], 2),
            (7, 5, {"counts": [3, 10, 22], "size": [7, 5]}, 3)]
    with torch.cuda.stream(side):                      # host inputs: the call itself must order its uploads before its kernels
        torch.cuda._sleep(SLEEP_CYCLES)
        planes, offs = cmask.rasterize(anns, cuda_dev)
    side.synchronize()
    host = planes.cpu().numpy().view(np.uint32)
    for i, (h, w, s, _) in enumerate(anns):
        assert np.array_equal(host[offs[i]:offs[i + 1]], ocm.pack(ocm.ann_mask(s, h, w))), i
    rng = np.random.RandomState(5)
    cases = [(37, 50, 4, 3), (1, 9, 2, 1), (64, 32, 3, 5)]
    preds = [rng.rand(M, h, w) < 0.4 for h, w, M, G in cases]
    gts = [rng.rand(G, h, w) < 0.3 for h, w, M, G in cases]
    up = lambda ms: _t(np.concatenate([m.reshape(-1).view(np.uint8) for m in ms]), cuda_dev)
    pack = lambda m, which: cmask.pack_masks(m, [(h, w, c[which]) for c in cases for h, w in [c[:2]]])
    want, pp = on_side(side, lambda m: pack(m, 2), [up(preds)], [1])
    assert_same(pp, want, "pack_masks")
    assert np.array_equal(pp.view(np.uint32), np.concatenate([ocm.pack(m) for p in preds for m in p]))
    gp = pack(up(gts), 3)
    want, got = on_side(side, lambda a, b: cmask.overlaps(a, b, cases), [_t(pp, cuda_dev), gp], [0, -1])
    assert_same(got, want, "overlaps")
    for (inter, ap, ag), p, g in zip(got, preds, gts):
        wi, wa, wg = ocm.overlaps(p, g)
        assert np.array_equal(inter, wi) and np.array_equal(ap, wa) and np.array_equal(ag, wg)


# ---------------------------------------------------------------------------------------------------------------- whole chain
def test_pipeline_on_a_side_stream(cuda_dev, side, cam_model):
    """run_u8 under a side stream (inputs late there) equals the default-stream labels; run() on host pyramids on that stream goes
    through the pipeline's copy stream, which then waits for a main stream that is not the default one."""
    from irn_b200.irn import EdgeDisplacement
    from irn_b200.pipeline import PseudoLabelPipeline, preprocess_batch
    irn = EdgeDisplacement()
    irn.load_state_dict(synth.irn_state_dict(), strict=False)
    H, W = 64, 80
    imgs = np.stack([synth.image(i, H, W) for i in range(2)])
    labels = torch.from_numpy(np.stack([synth.label(i) for i in range(2)]))
    pipe = PseudoLabelPipeline(cam_model, irn, cuda_dev, scales=(1.0, 0.5))
    f = lambda x: pipe.run_u8(x, labels, want_highres=False)["labels"]
    want, got = on_side(side, f, [_t(imgs, cuda_dev)], [0])
    assert_same(got, want, "run_u8")
    host = preprocess_batch(list(imgs), scales=(1.0, 0.5), pin=True)
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        out = pipe.run(host, labels, (H, W), want_highres=False)["labels"]
    side.synchronize()
    assert_same(_host(out), want, "run on host pyramids")


# ------------------------------------------------------------------------------------------------------- two streams, one cache
def _span(t):
    return t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()


def _overlap(a, b):
    return a[0] < b[1] and b[0] < a[1]


def test_workspace_and_scratch_are_per_stream(cuda_dev):
    a, b = torch.cuda.Stream(cuda_dev), torch.cuda.Stream(cuda_dev)
    for get in (lambda: indexing._workspace(1 << 20, cuda_dev), lambda: indexing._scratch(cuda_dev), lambda: cam_ops._scratch(cuda_dev)):
        with torch.cuda.stream(a):
            ta = get()
        with torch.cuda.stream(b):
            tb = get()
        assert not _overlap(_span(ta), _span(tb))
        with torch.cuda.stream(a):
            assert get().data_ptr() == ta.data_ptr()       # still cached for stream a


def test_growing_one_streams_workspace_keeps_anothers_queued_block(cuda_dev):
    """A walk queued on stream A behind a sleep; on stream B the cached workspace grows past A's block, then a walk runs.  A's block
    must not go back to the allocator while A's walk is pending: an allocation of its size on the default stream, where a cache
    shared by all streams would have allocated it, must not land on it; and both walks give their serial results."""
    a, b = torch.cuda.Stream(cuda_dev), torch.cuda.Stream(cuda_dev)
    h, w, C = 48, 40, 2
    x, e = synth.seeds(C, h, w, 1), synth.edge_map(h, w, "bimodal", 1)
    xb, eb = synth.seeds(8, 96, 96, 2), synth.edge_map(96, 96, "bimodal", 2)
    serial_a = indexing.random_walk_batch(_t(x, cuda_dev), _t(e, cuda_dev), [0, C], n_iter=32).cpu().numpy()
    indexing._workspace(indexing._workspace(0, cuda_dev).numel() + 1, cuda_dev)      # a fresh block cached on the default stream
    xa, ea = late(a, [_t(x, cuda_dev), _t(e, cuda_dev)], [NAN, NAN])
    with torch.cuda.stream(a):
        out_a = indexing.random_walk_batch(xa, ea, [0, C], n_iter=32)
        span_a = _span(indexing._workspace(0, cuda_dev))
    xb_d, eb_d = _t(xb, cuda_dev), _t(eb, cuda_dev)
    b.wait_stream(torch.cuda.default_stream(cuda_dev))
    with torch.cuda.stream(b):
        grown = indexing._workspace(2 * (span_a[1] - span_a[0]), cuda_dev)      # more than A's block holds, whatever is cached
        out_b = indexing.random_walk_batch(xb_d, eb_d, [0, 8], n_iter=32)
    assert not _overlap(_span(grown), span_a)
    reuse = torch.empty(span_a[1] - span_a[0], dtype=torch.uint8, device=cuda_dev)     # default stream
    assert not _overlap(_span(reuse), span_a), "stream A's queued workspace went back to the allocator"
    a.synchronize()
    b.synchronize()
    assert_same(_host(out_a), serial_a, "stream A")
    serial_b = indexing.random_walk_batch(xb_d, eb_d, [0, 8], n_iter=32).cpu().numpy()
    assert_same(_host(out_b), serial_b, "stream B")


def _gate(dev):
    """An event that completes after a sleep on a stream of its own: work on other streams that waits for it starts together."""
    g = torch.cuda.Stream(dev)
    with torch.cuda.stream(g):
        torch.cuda._sleep(SLEEP_CYCLES)
        ev = torch.cuda.Event()
        ev.record(g)
    return ev


def test_rw_labels_on_two_streams_with_different_maxima(cuda_dev):
    rng = np.random.default_rng(11)
    C, h, w, H, W = 8, 128, 128, 512, 512
    r1 = rng.random((C, h, w)).astype(np.float32)
    r2 = 0.01 * rng.random((C, h, w)).astype(np.float32)          # a hundred times smaller maximum
    d1, d2 = _t(r1, cuda_dev), _t(r2, cuda_dev)
    s1 = _host(indexing.rw_labels(d1, None, (H, W), 0.25, want_index=True, want_scores=True))
    s2 = _host(indexing.rw_labels(d2, None, (H, W), 0.25, want_index=True, want_scores=True))
    a, b = torch.cuda.Stream(cuda_dev), torch.cuda.Stream(cuda_dev)
    ev = _gate(cuda_dev)
    outs = []
    for s, d in ((a, d1), (b, d2)):
        s.wait_stream(torch.cuda.default_stream(cuda_dev))
        s.wait_event(ev)
        with torch.cuda.stream(s):
            outs.append(indexing.rw_labels(d, None, (H, W), 0.25, want_index=True, want_scores=True))
    a.synchronize()
    b.synchronize()
    assert_same(_host(outs[0]), s1, "stream A")
    assert_same(_host(outs[1]), s2, "stream B")


def test_cam_and_irnet_forwards_on_two_streams_share_no_workspace(cuda_dev, cam_model, irn_model):
    """A CAM forward on A and an IRNet forward on B, both held back by one event and released together (their serial runs left
    a workspace cached on the default stream that would fit either): each equals its serial result."""
    xc = _t(_pair(synth.image(1, 64, 80)), cuda_dev)
    xi = _t(_pair(synth.image(2, 128, 128)), cuda_dev)
    serial_c = _host(cam_model.forward_batch(xc))
    serial_i = _host(irn_model.forward_batch(xi))
    a, b = torch.cuda.Stream(cuda_dev), torch.cuda.Stream(cuda_dev)
    ev = _gate(cuda_dev)
    for s in (a, b):
        s.wait_stream(torch.cuda.default_stream(cuda_dev))
        s.wait_event(ev)
    with torch.cuda.stream(a):
        out_c = cam_model.forward_batch(xc)
    with torch.cuda.stream(b):
        out_i = irn_model.forward_batch(xi)
    a.synchronize()
    b.synchronize()
    assert_same(_host(out_c), serial_c, "CAM on stream A")
    assert_same(_host(out_i), serial_i, "IRNet on stream B")


# ---------------------------------------------------------------------------------------------------- two host threads, two streams
def test_two_host_threads_two_streams(cuda_dev):
    """Thread 1 walks at radius 5 (fused); thread 2 computes affinities at radius 3 and 10 and walks at radius 3 (generic kernel),
    so the radius tables switch while thread 1 walks.  Each then runs rw_labels and a CRF.  Every result equals the serial one, and
    the error text, the last-walk flag and the timing switch of one thread are not the other's."""
    L = _lib.lib()
    h, w, C = 64, 64, 3
    x, e = synth.seeds(C, h, w, 3), synth.edge_map(h, w, "bimodal", 3)
    e3 = synth.edge_map(37, 45, "uniform", 3)
    img = synth.image(4, 24, 28)
    lab = synth.cam_planes_u8(3, 24, 28, 4).argmax(0).astype(np.int32)

    def t1_work():
        rw = indexing.random_walk_batch(_t(x, cuda_dev), _t(e, cuda_dev), [0, C], 5, 10, 64, variant=4)
        fused = indexing.last_walk_was_fused()
        labels = indexing.rw_labels(rw, [1, 4, 9], (4 * h - 3, 4 * w - 1))[0]
        q = crf.dense_crf(_t(img[None], cuda_dev), _t(lab[None], cuda_dev), 3, want_q=True)
        return _host((rw, labels, q)), fused

    def t2_work():
        a3 = indexing.edge_to_affinity(_t(e3, cuda_dev), 3)
        a10 = indexing.edge_to_affinity(_t(e3, cuda_dev), 10)
        rw = indexing.random_walk_batch(_t(x, cuda_dev), _t(e, cuda_dev), [0, C], 3, 10, 64, variant=1)
        fused = indexing.last_walk_was_fused()
        labels = indexing.rw_labels(rw, None, (4 * h, 4 * w), want_index=True)
        q = crf.dense_crf(_t(img[None], cuda_dev), _t(1 - np.minimum(lab, 1)[None], cuda_dev), 2, want_q=True)
        return _host((a3, a10, rw, labels, q)), fused

    serial = [t1_work(), t2_work()]
    assert serial[0][1] and not serial[1][1]
    results, errors = [None, None], []
    barrier = threading.Barrier(2, timeout=120)

    def run(i):
        try:
            s = torch.cuda.Stream(cuda_dev)
            with torch.cuda.stream(s):
                # per-thread state: thread 1 switches walk timing on and leaves an error; thread 2 then leaves another error
                if i == 0:
                    L.irn_rw_set_timing(1)
                    assert L.irn_random_walk_variant(None, None, None, 1, None, 8, 8, 5, 10.0, 1, None, 0, 3, None) != 0
                    msg = L.irn_last_error()
                    assert b"unknown variant" in msg
                barrier.wait()
                if i == 1:
                    assert L.irn_random_walk_variant(None, None, None, 1, None, 8, 8, 5, 10.0, 1, None, 0, 1, None) != 0
                    assert b"null pointer" in L.irn_last_error()
                barrier.wait()
                if i == 0:
                    assert L.irn_last_error() == msg, "thread 2's error reached thread 1"
                # both threads at once: thread 2's radius switches happen while thread 1 walks at radius 5
                res = t1_work() if i == 0 else t2_work()
                s.synchronize()
                if i == 0:
                    ms, n = ctypes.c_float(), ctypes.c_int()
                    assert L.irn_rw_last_step_ms(ctypes.byref(ms), ctypes.byref(n)) == 0 and n.value == 64
                    L.irn_rw_set_timing(0)
                else:
                    assert L.irn_rw_last_step_ms(ctypes.byref(ctypes.c_float()), None) != 0, "thread 1's timing switch reached thread 2"
                results[i] = res
        except BaseException as ex:          # re-raised by the main thread
            errors.append(ex)
            barrier.abort()

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    assert_same(results[0], serial[0], "thread 1")
    assert_same(results[1], serial[1], "thread 2")
    W3, _ = oi.stencil_weights(e3, 3, beta=1)
    W10, _ = oi.stencil_weights(e3, 10, beta=1)
    assert np.array_equal(results[1][0][0][0], W3) and np.array_equal(results[1][0][1][0], W10)
