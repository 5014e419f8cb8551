"""Batches of images of different sizes through IRNet and the random walk, bit for bit against the one-size paths.

EdgeDisplacement.forward_ragged runs every image on the zero-padded crop_size canvas (as the reference pads each one,
net/resnet50_irn.py:226); each image's corner of its output must equal forward_batch of that image alone, with edge 1.0 / dp 0
outside.  The walk on such a padded grid must equal the walk on the image's own grid, and the size-agnostic steps must write the same
files as the one-image loop on a list of mixed sizes."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch
from PIL import Image

from irn_b200 import _lib, indexing, preprocess, synth
from irn_b200.irn import EdgeDisplacement, _normalize_lut

pytestmark = pytest.mark.gpu

SIZES = [(512, 512), (500, 375), (375, 500), (333, 500), (61, 97), (1, 1), (2, 3)]


@pytest.fixture(scope="module")
def irn_model(cuda_dev):
    m = EdgeDisplacement()
    m.load_state_dict(synth.irn_state_dict(), strict=False)
    m.eval()
    return m


@pytest.fixture(scope="module")
def images(cuda_dev):
    return [torch.from_numpy(synth.image(40 + i, h, w)).to(cuda_dev) for i, (h, w) in enumerate(SIZES)]


def _single(model, img):
    """forward_batch of one image: the scale-1.0 (image, flipped image) pair of the device loader."""
    x = preprocess.msf_batch(img[None], (1.0,))[0]
    e, d = model.forward_batch(x)
    return e[0], d[0]


def _check(edge, dp, refs, order):
    fc = edge.shape[-1]
    for i, k in enumerate(order):
        h, w = SIZES[k]
        fh, fw = (h - 1) // 4 + 1, (w - 1) // 4 + 1
        e_ref, d_ref = refs[k]
        assert torch.equal(edge[i, :, :fh, :fw], e_ref), (SIZES[k], "edge")
        assert torch.equal(dp[i, :, :fh, :fw], d_ref), (SIZES[k], "dp")
        pad_e = torch.ones((1, fc, fc), device=edge.device)
        pad_e[:, :fh, :fw] = e_ref
        assert torch.equal(edge[i], pad_e), (SIZES[k], "edge pad is not 1.0")
        pad_d = torch.zeros((2, fc, fc), device=dp.device)
        pad_d[:, :fh, :fw] = d_ref
        assert torch.equal(dp[i], pad_d), (SIZES[k], "dp pad is not 0")


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_ragged_forward_equals_forward_batch_per_image(irn_model, images, mode):
    irn_model.set_conv_mode(mode)
    try:
        refs = [_single(irn_model, img) for img in images]
        n = len(images)
        shuffled = [int(i) for i in np.random.default_rng(mode).permutation(n)]
        for order in ([1], [0, 4, 5], list(range(n)), shuffled):
            edge, dp = irn_model.forward_ragged([images[k] for k in order])
            fc = (irn_model.crop_size - 1) // 4 + 1
            assert edge.shape == (len(order), 1, fc, fc) and dp.shape == (len(order), 2, fc, fc)
            _check(edge, dp, refs, order)
        # the packed form: one flat buffer and the sizes
        order = shuffled[:3]
        flat = torch.cat([images[k].reshape(-1) for k in order])
        edge, dp = irn_model.forward_ragged(flat, [SIZES[k] for k in order])
        _check(edge, dp, refs, order)
    finally:
        irn_model.set_conv_mode(None)


def _pad(t, fh, fw, value):
    out = torch.full(t.shape[:-2] + (fh, fw), value, dtype=t.dtype, device=t.device)
    out[..., :t.shape[-2], :t.shape[-1]] = t
    return out


@pytest.mark.parametrize("exp_times", [0, 8])
@pytest.mark.parametrize("v_own,v_pad", [(2, 2), (4, 4), (2, 4), (4, 2), (0, 0)])
def test_walk_on_padded_grid_equals_walk_on_own_grid(cuda_dev, v_own, v_pad, exp_times):
    grids = [(125, 94), (94, 125), (16, 25), (1, 1), (128, 128), (7, 3)]
    channels = [1, 3, 2, 5, 4, 21]
    kinds = ["bimodal", "uniform", "low", "sigmoid4", "bimodal", "uniform"]
    edges, seeds = [], []
    for i, ((h, w), c, kind) in enumerate(zip(grids, channels, kinds)):
        edges.append(torch.from_numpy(synth.edge_map(h, w, kind, 70 + i)).to(cuda_dev))
        seeds.append(torch.from_numpy(synth.seeds(c, h, w, 70 + i)).to(cuda_dev))
    n_iter = 2 ** exp_times
    own = [indexing.random_walk_batch(s, e, [0, s.shape[0]], 5, 10, n_iter, variant=v_own) for s, e in zip(seeds, edges)]
    fc = 128
    pe = torch.cat([_pad(e, fc, fc, 1.0) for e in edges], 0)
    ps = torch.cat([_pad(s, fc, fc, 0.0) for s in seeds], 0)
    offs = np.concatenate([[0], np.cumsum(channels)])
    walk = indexing.random_walk_batch(ps, pe, offs, 5, 10, n_iter, variant=v_pad)
    for i, ((h, w), r) in enumerate(zip(grids, own)):
        assert torch.equal(walk[offs[i]:offs[i + 1], :h, :w], r), (grids[i], "in-image")
        assert not walk[offs[i]:offs[i + 1]].isnan().any()


def test_ragged_forward_rejects_bad_input(irn_model, images, cuda_dev):
    L = _lib.lib()
    plan = irn_model._get_plan(cuda_dev)
    S = irn_model.crop_size
    fc = (S - 1) // 4 + 1
    img = images[4].reshape(-1).contiguous()
    lut = _normalize_lut(cuda_dev)
    edge = torch.empty((1, 1, fc, fc), device=cuda_dev)
    dp = torch.empty((1, 2, fc, fc), device=cuda_dev)
    need = L.irn_edge_displacement_ragged_workspace_bytes(1, S)
    ws = torch.empty(need + 512, dtype=torch.uint8, device=cuda_dev)
    host_img = np.zeros(img.numel(), np.uint8)

    def call(hw, off=0, src=None, ws_ptr=None, ws_bytes=need, table=None):
        hw = np.ascontiguousarray(np.asarray(hw, np.int32).reshape(1, 2))
        offs = np.array([off], np.int64)
        src = _lib.ptr(img) if src is None else src
        ws_ptr = _lib.ptr(ws) if ws_ptr is None else ws_ptr
        table = _lib.ptr(lut) if table is None else table
        with torch.cuda.device(cuda_dev):
            return L.irn_edge_displacement_forward_ragged(plan.handle, src, img.numel(), offs.ctypes.data, hw.ctypes.data, 1, S, table,
                                                          _lib.ptr(edge), _lib.ptr(dp), ws_ptr, ws_bytes, _lib.stream_ptr())

    assert call((61, 97)) == 0
    torch.cuda.synchronize()
    assert call((0, 97)) == -1
    assert call((61, -1)) == -1
    assert call((S + 1, 97)) == -1
    assert call((61, 97), off=1) == -1                                   # runs past the end of the image buffer
    assert call((61, 97), off=-3) == -1
    assert call((61, 97), src=ctypes.c_void_p(host_img.ctypes.data)) == -1     # host memory
    assert call((61, 97), table=ctypes.c_void_p(preprocess.normalize_lut().ctypes.data)) == -1
    assert call((61, 97), ws_ptr=ctypes.c_void_p(ws.data_ptr() + 16)) == -1      # misaligned workspace
    assert call((61, 97), ws_bytes=need - 256) == -3
    assert b"workspace" in L.irn_last_error()
    with pytest.raises(_lib.IrnError):
        irn_model.forward_ragged([images[0][:, :, :2]])                  # not RGB-sized: the byte count disagrees
    with pytest.raises(_lib.IrnError):
        irn_model.forward_ragged(img.float(), [(61, 97)])
    with pytest.raises(_lib.IrnError):
        irn_model.forward_ragged(torch.zeros((S + 4) * 8 * 3, dtype=torch.uint8, device=cuda_dev), [(S + 4, 8)])
    # nothing above faulted: the device still runs the forward and gives the same answer
    e2, d2 = irn_model.forward_ragged([images[4]])
    assert call((61, 97)) == 0
    torch.cuda.synchronize()
    assert torch.equal(edge, e2) and torch.equal(dp, d2)


# ------------------------------------------------------------------ the steps on a list of mixed sizes

MIXED = [(64, 96), (96, 64), (77, 50), (512, 512)]


def _same_tree(a_dir, b_dir, names, kind):
    for n in names:
        if kind == "png":
            a = np.asarray(Image.open(os.path.join(a_dir, n + ".png")))
            b = np.asarray(Image.open(os.path.join(b_dir, n + ".png")))
            assert a.shape == b.shape and np.array_equal(a, b), n
            continue
        a = np.load(os.path.join(a_dir, n + ".npy"), allow_pickle=True).item()
        b = np.load(os.path.join(b_dir, n + ".npy"), allow_pickle=True).item()
        assert set(a) == set(b)
        for k in a:
            x, y = (v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v) for v in (a[k], b[k]))
            # raw bytes: a score can be NaN (a detection over an all-zero walk), and the same NaN must come out of both runs
            assert type(a[k]) is type(b[k]) and x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (n, k)


def test_mixed_size_steps_write_the_same_files(cuda_dev, tmp_path):
    """make_cam, make_sem_seg_labels and make_ins_seg_labels on a list mixing four sizes: --step_batch 4 (size buckets for make_cam,
    batches of any sizes for the label steps) writes the same files, byte for byte, as --step_batch 1 (the reference's loop)."""
    from irn_b200.step import _common, make_cam, make_ins_seg_labels, make_sem_seg_labels
    from irn_b200.voc12 import dataloader
    n = 10
    names = ["2007_%06d" % i for i in range(n)]
    os.makedirs(tmp_path / "sess")
    torch.save(synth.cam_state_dict(), tmp_path / "sess" / "res50_cam.pth.pth")
    torch.save(synth.irn_state_dict(), tmp_path / "sess" / "res50_irn.pth")
    real = _common.make_dataset

    def mixed(a, list_path, scales, cam_dir=None):
        if _common.step_batch(a) == 1:
            cam_dir = None          # the one-image loop reads the stored CAMs itself, like the reference
        return dataloader.SyntheticMSF(n, scales=scales, decode_only=_common.device_pyramid(a), cam_dir=cam_dir, sizes=MIXED)

    runs = []
    _common.make_dataset = mixed
    try:
        for tag, bsz in (("b1", 1), ("b4", 4)):
            a = types.SimpleNamespace(
                num_workers=0, voc12_root=str(tmp_path), train_list="", infer_list="", cam_network="irn_b200.cam",
                irn_network="irn_b200.irn", cam_scales=(1.0, 0.5, 1.5, 2.0), cam_weights_name=str(tmp_path / "sess" / "res50_cam.pth"),
                irn_weights_name=str(tmp_path / "sess" / "res50_irn.pth"), beta=10, exp_times=5, sem_seg_bg_thres=0.25,
                ins_seg_bg_thres=0.25, synthetic=n, step_batch=bsz)
            for k in ("cam_out_dir", "sem_seg_out_dir", "ins_seg_out_dir"):
                d = tmp_path / (tag + "_" + k)
                os.makedirs(d)
                setattr(a, k, str(d))
            make_cam.run(a)
            make_sem_seg_labels.run(a)
            make_ins_seg_labels.run(a)
            runs.append(a)
    finally:
        _common.make_dataset = real
    one, many = runs
    _same_tree(one.cam_out_dir, many.cam_out_dir, names, "npy")
    _same_tree(one.sem_seg_out_dir, many.sem_seg_out_dir, names, "png")
    _same_tree(one.ins_seg_out_dir, many.ins_seg_out_dir, names, "npy")
    for i, name in enumerate(names):
        assert np.asarray(Image.open(os.path.join(many.sem_seg_out_dir, name + ".png"))).shape == MIXED[i % len(MIXED)]
