"""The CAM stage on batches of images of different sizes, bit for bit against the one-size paths.

CAM.forward_ragged runs (image, flipped image) pairs of different sizes on one canvas, each at the top-left corner; the trunk zeroes
the padding of the tensors its spatial operators read beyond an image's extent, so each pair's corner of the output must equal
forward_batch of that pair alone, in every conv mode, with 0 elsewhere.  The ragged pyramid must equal resize_normalize per image with
+0.0 padding, cam_ragged_stage must equal cam_stage per image, and make_cam with size buckets topped up by smaller images must write
the same files as the one-image loop."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from irn_b200 import _lib, preprocess, synth
from irn_b200.cam import CAM
from irn_b200.irn import _normalize_lut
from irn_b200.pipeline import PseudoLabelPipeline

pytestmark = pytest.mark.gpu

# every residue class of an extent at each stride level (2, 4, 8, 16), both orientations, the largest canvas last
SIZES = [(1, 1), (2, 3), (17, 33), (61, 97), (333, 500), (375, 500), (500, 375), (512, 512)]
SCALES = (1.0, 0.5, 1.5, 2.0)


@pytest.fixture(scope="module")
def cam_model(cuda_dev):
    m = CAM()
    m.load_state_dict(synth.cam_state_dict(), strict=True)
    m.eval()
    return m


@pytest.fixture(scope="module")
def images(cuda_dev):
    return [torch.from_numpy(synth.image(60 + i, h, w)).to(cuda_dev) for i, (h, w) in enumerate(SIZES)]


def _valid(scale, order):
    """The images of `order` that still have a pixel at `scale` (1x1 rounds to 0x0 at 0.5, for the reference's loader too)."""
    return [k for k in order if min(preprocess.rescaled_size(*SIZES[k], scale)) > 0]


def _flat(images, order):
    return torch.cat([images[k].reshape(-1) for k in order])


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("scale", SCALES)
def test_ragged_pyramid_equals_resize_normalize_per_image(images, scale):
    order = _valid(scale, [int(i) for i in np.random.default_rng(int(scale * 10)).permutation(len(SIZES))])
    canvas, ext = preprocess.resize_normalize_ragged(_flat(images, order), [SIZES[k] for k in order], scale)
    Hc, Wc = max(h for h, _ in ext), max(w for _, w in ext)
    assert canvas.shape == (2 * len(order), 3, Hc, Wc) and canvas.dtype == torch.float32
    for i, k in enumerate(order):
        H, W = SIZES[k]
        assert ext[i] == ((H, W) if scale == 1 else preprocess.rescaled_size(H, W, scale))
        ref = preprocess.resize_normalize(images[k][None], ext[i])
        want = torch.zeros((2, 3, Hc, Wc), device=canvas.device)
        want[:, :, :ext[i][0], :ext[i][1]] = ref
        # bitwise, so the padding is +0.0, not -0.0
        assert torch.equal(_bits(canvas[2 * i:2 * i + 2]), _bits(want)), (SIZES[k], scale)


def _cam_ref(model, img, scale):
    """forward_batch of one image's (image, flipped image) pair at `scale`, the one-size path."""
    return model.forward_batch(preprocess.msf_batch(img[None], (scale,))[0])[0]


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_forward_ragged_equals_forward_batch_per_image(cam_model, images, mode):
    cam_model.set_conv_mode(mode)
    try:
        n = len(SIZES)
        shuffled = [int(i) for i in np.random.default_rng(mode).permutation(n)]
        for scale in SCALES:
            refs = {k: _cam_ref(cam_model, images[k], scale) for k in _valid(scale, range(n))}
            assert any(r.abs().max() > 0 for r in refs.values())
            for order in (_valid(scale, shuffled), [2], _valid(scale, [7, 0, 3])):
                canvas, ext = preprocess.resize_normalize_ragged(_flat(images, order), [SIZES[k] for k in order], scale)
                out = cam_model.forward_ragged(canvas, ext)
                Hc, Wc = canvas.shape[-2:]
                hc, wc = (Hc - 1) // 16 + 1, (Wc - 1) // 16 + 1
                assert out.shape == (len(order), 20, hc, wc)
                for i, k in enumerate(order):
                    h, w = refs[k].shape[-2:]
                    assert (h, w) == ((ext[i][0] - 1) // 16 + 1, (ext[i][1] - 1) // 16 + 1)
                    want = torch.zeros((20, hc, wc), device=out.device)
                    want[:, :h, :w] = refs[k]
                    assert torch.equal(out[i], want), (SIZES[k], scale, mode, order)
    finally:
        cam_model.set_conv_mode(None)


def test_cam_ragged_stage_equals_cam_stage_per_image(cam_model, images, cuda_dev):
    rng = np.random.default_rng(5)
    labels = torch.from_numpy((rng.random((len(SIZES), 20)) < 0.2).astype(np.float32))
    labels[1] = 0                       # an image without a class
    labels[2, 3] = 1
    # cam_sub_batch 1: at scale 2.0 every image is a forward of its own, at 0.5 all eight share one
    pipe = PseudoLabelPipeline(cam_model, None, cuda_dev, SCALES, cam_sub_batch=1)
    order = [int(i) for i in rng.permutation(len(SIZES)) if SIZES[i] != (1, 1)]
    keys, strided, highres = pipe.cam_ragged_stage(_flat(images, order), [SIZES[k] for k in order], labels[order])
    assert len(keys) == len(strided) == len(highres) == len(order)
    for i, k in enumerate(order):
        H, W = SIZES[k]
        rk, rs, rh = pipe.cam_stage(pipe.pyramids(images[k][None]), labels[k:k + 1], (H, W))
        assert np.array_equal(keys[i], rk[0]), SIZES[k]
        assert strided[i].shape == rs[0].shape and torch.equal(strided[i], rs[0]), SIZES[k]
        assert highres[i].shape == rh[0].shape == (len(rk[0]), H, W) and torch.equal(highres[i], rh[0]), SIZES[k]


def test_ragged_entry_points_reject_bad_input(cam_model, images, cuda_dev):
    L = _lib.lib()
    plan = cam_model._get_plan(cuda_dev)
    order = [3, 2]
    flat = _flat(images, order)
    canvas, ext = preprocess.resize_normalize_ragged(flat, [SIZES[k] for k in order], 1.0)
    B, _, Hc, Wc = canvas.shape
    out = torch.empty((B // 2, 20, (Hc - 1) // 16 + 1, (Wc - 1) // 16 + 1), device=cuda_dev)
    need = L.irn_cam_workspace_bytes(B, Hc, Wc)
    ws = torch.empty(need + 512, dtype=torch.uint8, device=cuda_dev)
    host_canvas = torch.zeros(canvas.shape)
    dev_hw = torch.tensor(ext, dtype=torch.int32, device=cuda_dev)

    def cam(hw=ext, b=B, x=None, ws_ptr=None, ws_bytes=need, hw_ptr=None):
        a = np.ascontiguousarray(np.asarray(hw, np.int32).reshape(-1, 2))
        with torch.cuda.device(cuda_dev):
            return L.irn_cam_forward_ragged(plan.handle, _lib.ptr(canvas) if x is None else x, b, Hc, Wc,
                                            a.ctypes.data if hw_ptr is None else hw_ptr, _lib.ptr(out),
                                            _lib.ptr(ws) if ws_ptr is None else ws_ptr, ws_bytes, _lib.stream_ptr())

    assert cam() == 0
    torch.cuda.synchronize()
    good = out.clone()
    assert cam(hw=[(61, 97), (0, 33)]) == -1
    assert cam(hw=[(61, 97), (17, -1)]) == -1
    assert cam(hw=[(Hc + 1, 97), (17, 33)]) == -1
    assert cam(hw=[(61, Wc + 1), (17, 33)]) == -1
    assert cam(b=3) == -1                                                      # odd B
    assert cam(x=ctypes.c_void_p(host_canvas.data_ptr())) == -1                # host canvas
    assert cam(hw_ptr=ctypes.c_void_p(dev_hw.data_ptr())) == -1                # extents in device memory
    assert cam(ws_ptr=ctypes.c_void_p(ws.data_ptr() + 16)) == -1               # misaligned workspace
    assert cam(ws_bytes=need - 256) == -3
    assert b"workspace" in L.irn_last_error()
    with pytest.raises(_lib.IrnError):
        cam_model.forward_ragged(canvas, ext[:1])                              # one extent for two pairs

    hw = np.ascontiguousarray(np.asarray([SIZES[k] for k in order], np.int32))
    offs = np.array([0, 3 * SIZES[3][0] * SIZES[3][1]], np.int64)
    rs_ws = torch.empty(L.irn_resize_ragged_workspace_bytes(hw.ctypes.data, hw.ctypes.data, 2) + 512, dtype=torch.uint8, device=cuda_dev)
    lut = _normalize_lut(cuda_dev)
    host_img = np.zeros(flat.numel(), np.uint8)

    def resize(ohw=hw, off=offs, src=None, hc=Hc, wc=Wc, p=2):
        o = np.ascontiguousarray(np.asarray(ohw, np.int32))
        off = np.ascontiguousarray(np.asarray(off, np.int64))
        with torch.cuda.device(cuda_dev):
            return L.irn_resize_ragged_forward(_lib.ptr(flat) if src is None else src, flat.numel(), off.ctypes.data, hw.ctypes.data,
                                               o.ctypes.data, p, hc, wc, _lib.ptr(lut), _lib.ptr(canvas), _lib.ptr(rs_ws), rs_ws.numel(),
                                               _lib.stream_ptr())

    assert resize() == 0
    torch.cuda.synchronize()
    assert resize(hc=Hc - 1) == -1                                             # an image larger than the canvas
    assert resize(ohw=[(61, 97), (0, 33)]) == -1
    assert resize(off=[0, flat.numel() - 3]) == -1                             # runs past the end of the image buffer
    assert resize(off=[-3, 0]) == -1
    assert resize(src=ctypes.c_void_p(host_img.ctypes.data)) == -1             # host images
    assert resize(p=0) == -1
    assert L.irn_resize_ragged_workspace_bytes(hw.ctypes.data, np.zeros((2, 2), np.int32).ctypes.data, 2) == 0
    with pytest.raises(_lib.IrnError):
        preprocess.resize_normalize_ragged(flat.float(), [SIZES[k] for k in order], 1.0)
    # nothing above faulted: the device still runs both and gives the same answer
    assert cam() == 0
    torch.cuda.synchronize()
    assert torch.equal(out, good)


# ------------------------------------------------------------------ make_cam on a list of many sizes

MIXED = [(64, 96), (60, 90), (64, 80), (56, 96), (48, 96), (96, 64), (90, 60), (80, 64), (33, 47), (30, 40), (17, 33),
         (100, 120), (90, 110), (75, 100)]


def test_make_cam_with_riders_writes_the_same_files(cuda_dev, tmp_path, monkeypatch):
    """make_cam on 42 images of 14 sizes: with --step_batch 4 the pending buckets pass the bound, and buckets flushed early or at the
    end take smaller images along (mixed batches through cam_ragged_stage); every entry of the .npy files is byte for byte that of
    --step_batch 1 (the reference's loop)."""
    from irn_b200.step import _common, make_cam
    from irn_b200.voc12 import dataloader
    n = 42
    names = ["2007_%06d" % i for i in range(n)]
    os.makedirs(tmp_path / "sess")
    torch.save(synth.cam_state_dict(), tmp_path / "sess" / "res50_cam.pth.pth")
    monkeypatch.setattr(_common, "make_dataset", lambda a, list_path, scales, cam_dir=None: dataloader.SyntheticMSF(
        n, scales=scales, decode_only=_common.device_pyramid(a), sizes=MIXED))
    batches = []
    real_batch = make_cam.cam_batch

    def recording(ctx, packs):
        batches.append([p["size"] for p in packs])
        return real_batch(ctx, packs)
    monkeypatch.setattr(make_cam, "cam_batch", recording)
    dirs = []
    for bsz in (1, 4):
        d = tmp_path / ("cam_b%d" % bsz)
        os.makedirs(d)
        make_cam.run(types.SimpleNamespace(num_workers=0, voc12_root=str(tmp_path), train_list="", cam_network="irn_b200.cam",
                                           cam_scales=SCALES, cam_weights_name=str(tmp_path / "sess" / "res50_cam.pth"), synthetic=n,
                                           step_batch=bsz, cam_out_dir=str(d)))
        dirs.append(d)
    assert sorted(s for b in batches for s in b) == sorted(MIXED[i % len(MIXED)] for i in range(n))
    assert any(len(set(b)) > 1 for b in batches), "no batch took a rider"
    for name in names:
        a = np.load(os.path.join(dirs[0], name + ".npy"), allow_pickle=True).item()
        b = np.load(os.path.join(dirs[1], name + ".npy"), allow_pickle=True).item()
        assert set(a) == set(b) == {"keys", "cam", "high_res"}
        for k in a:
            x, y = (v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v) for v in (a[k], b[k]))
            assert type(a[k]) is type(b[k]) and x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (name, k)
