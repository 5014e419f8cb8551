"""The exact JPEG decoder on the device (irn_b200.jpeg.ExactJpegDecoder, csrc/jpeg_exact.cu) bit for bit against PIL's pixels in
tests/golden/jpeg_exact.npz and against the oracle (oracle/jpeg.py); ragged calls, batch invariance, corrupt entropy-coded data;
and the steps with --device_jpeg exact writing the same files as with the host decoder."""
import io
import os
import types

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import golden_path
from irn_b200 import _lib, synth
from oracle import jpeg as oracle_jpeg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cases():
    g = np.load(golden_path("jpeg_exact.npz"))
    return [(str(g["name%d" % i]), g["jpeg%d" % i].tobytes(), g["pixels%d" % i]) for i in range(int(g["n"]))]


@pytest.fixture(scope="module")
def dec(cuda_dev):
    from irn_b200.jpeg import ExactJpegDecoder
    return ExactJpegDecoder(cuda_dev)


def test_every_case_equals_pil_and_oracle(cases, dec):
    for name, data, pixels in cases:
        got = dec.decode([data], names=[name])
        assert got.shape == (1,) + pixels.shape and got.dtype == torch.uint8, name
        got = got[0].cpu().numpy()
        assert np.array_equal(got, pixels), (name, int(np.abs(got.astype(int) - pixels).max()))
        assert np.array_equal(got, oracle_jpeg.decode(data)), name


def _split(flat, sizes):
    out, o = [], 0
    flat = flat.cpu().numpy()
    for h, w in sizes:
        out.append(flat[o:o + 3 * h * w].reshape(h, w, 3))
        o += 3 * h * w
    return out


def test_ragged_call_equals_per_image_calls(cases, dec):
    flat, sizes = dec.decode_packed([d for _, d, _ in cases], names=[n for n, _, _ in cases])
    assert sizes == [p.shape[:2] for _, _, p in cases]
    assert flat.numel() == sum(p.size for _, _, p in cases)
    for (name, data, pixels), got in zip(cases, _split(flat, sizes)):
        assert np.array_equal(got, dec.decode([data])[0].cpu().numpy()), name
        assert np.array_equal(got, pixels), name


def test_batch_invariant_and_deterministic(cases, dec):
    rng = np.random.default_rng(5)
    order = [int(i) for i in rng.permutation(len(cases))]
    streams = [cases[i][1] for i in order]
    a, sizes = dec.decode_packed(streams)
    b, _ = dec.decode_packed(streams)
    assert torch.equal(a, b)
    for i, got in zip(order, _split(a, sizes)):
        assert np.array_equal(got, cases[i][2]), cases[i][0]
    # one size, [n,H,W,3]; every image alone and inside batches of other compositions
    same = [c for c in cases if c[2].shape == (40, 56, 3)]
    out = dec.decode([d for _, d, _ in same]).cpu().numpy()
    for k, (name, _, pixels) in enumerate(same):
        assert np.array_equal(out[k], pixels), name
    sub, _ = dec.decode_packed([same[3][1], cases[-1][1], same[0][1]])
    assert np.array_equal(_split(sub, [(40, 56), cases[-1][2].shape[:2], (40, 56)])[2], same[0][2])


def _corrupt_cases():
    img = synth.image(11, 64, 80)
    b = io.BytesIO()
    Image.fromarray(img).save(b, format="JPEG", quality=90)
    plain = b.getvalue()
    b = io.BytesIO()
    Image.fromarray(img).save(b, format="JPEG", quality=90, restart_marker_blocks=2)
    rst = b.getvalue()
    s0 = plain.index(b"\xff\xda")
    s0 += 2 + (plain[s0 + 2] << 8 | plain[s0 + 3])
    r0 = rst.index(b"\xff\xd0")
    return {
        "ends early": plain[:s0 + 40] + b"\xff\xd9",                          # valid headers, entropy data cut short
        "stray marker": plain[:s0 + 60] + b"\xff\xc4" + plain[s0 + 60:],      # a marker inside the scan
        "missing restart": rst[:r0] + rst[r0 + 2:],                           # one RSTn dropped
        "garbage": plain[:s0] + bytes([0xFF, 0x00] * 300) + b"\xff\xd9",      # all-ones bits: no valid Huffman code
    }, plain


def test_corrupt_entropy_data_raises_through_the_status_word(dec):
    bad, good = _corrupt_cases()
    want = dec.decode([good])[0]
    for what, data in bad.items():
        assert oracle_jpeg.inspect(data)[:2] == (64, 80)       # the headers are fine: only the device can tell
        with pytest.raises(_lib.IrnError, match="bad_%s" % what.replace(" ", "_")):
            dec.decode([good, data], names=["good", "bad_%s" % what.replace(" ", "_")])
        out, st = dec.decode([good, data], check=False)
        torch.cuda.synchronize()
        assert int(st.status[0]) == 0 and int(st.status[1]) != 0, what
        assert torch.equal(out[0], want), what


# ---------------------------------------------------------------------------------------------------------------------------------
# the steps with --device_jpeg exact against the host decoder

@pytest.fixture(scope="module")
def voc_tree(tmp_path_factory, cuda_dev):
    """JPEG files of mixed sizes (the reference-run images of tests/golden/steps.npz and synthetic ones, 4:2:0 and 4:4:4), one PNG
    stand-in and one progressive JPEG (both decoded on the host by the loader in the exact runs, mixed into the same batches)."""
    g = np.load(golden_path("steps.npz"))
    root = tmp_path_factory.mktemp("voc_exact")
    os.makedirs(root / "JPEGImages")
    labels, ids = {}, []

    def add(name, img, label, **kw):
        Image.fromarray(img).save(root / "JPEGImages" / (name + ".jpg"), **kw)
        labels[int(name.replace("_", ""))] = label
        ids.append(name)
    for i, name in enumerate(str(s) for s in g["ids"]):
        add(name, g["img%d" % i], g["label%d" % i], quality=95)
    add("2008_000001", synth.image(81, 96, 128), synth.label(1, 2), quality=90, subsampling=0)
    add("2008_000002", synth.image(82, 96, 128), synth.label(2, 2), quality=85, optimize=True, restart_marker_blocks=5)
    add("2008_000003", synth.image(83, 96, 128), synth.label(3, 2), format="PNG")
    add("2008_000004", synth.image(84, 80, 112), synth.label(4, 2), quality=90)
    add("2008_000005", synth.image(85, 75, 100), synth.label(5, 2), quality=90, progressive=True)
    (root / "all.txt").write_text("\n".join(ids) + "\n")
    one = [n for n in ids if Image.open(root / "JPEGImages" / (n + ".jpg")).size == (128, 96)]
    (root / "one.txt").write_text("\n".join(one) + "\n")
    os.makedirs(root / "sess")
    torch.save(synth.cam_state_dict(), root / "sess" / "res50_cam.pth.pth")
    torch.save(synth.irn_state_dict(), root / "sess" / "res50_irn.pth")
    from irn_b200.voc12 import dataloader
    dataloader._cls_labels["voc12/cls_labels.npy"] = labels
    return root, ids, one


def _args(root, tag, lst, **over):
    a = types.SimpleNamespace(
        num_workers=0, voc12_root=str(root), train_list=str(root / lst), infer_list=str(root / lst), cam_network="irn_b200.cam",
        irn_network="irn_b200.irn", cam_scales=(1.0, 0.5, 1.5, 2.0), cam_weights_name=str(root / "sess" / "res50_cam.pth"),
        irn_weights_name=str(root / "sess" / "res50_irn.pth"), beta=10, exp_times=8, sem_seg_bg_thres=0.25, ins_seg_bg_thres=0.25,
        conf_fg_thres=0.30, conf_bg_thres=0.05, synthetic=0, step_batch=4)
    for k in ("cam_out_dir", "sem_seg_out_dir", "ins_seg_out_dir", "ir_label_out_dir"):
        d = root / (tag + "_" + k)
        os.makedirs(d, exist_ok=True)
        setattr(a, k, str(d))
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _same_npy(a_dir, b_dir, names):
    for n in names:
        a = np.load(os.path.join(a_dir, n + ".npy"), allow_pickle=True).item()
        b = np.load(os.path.join(b_dir, n + ".npy"), allow_pickle=True).item()
        assert set(a) == set(b), n
        for k in a:
            x, y = (v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v) for v in (a[k], b[k]))
            # bitwise (a detection score can be NaN in both runs)
            assert type(a[k]) is type(b[k]) and x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (n, k)


def _same_png(a_dir, b_dir, names):
    for n in names:
        with open(os.path.join(a_dir, n + ".png"), "rb") as f, open(os.path.join(b_dir, n + ".png"), "rb") as h:
            assert f.read() == h.read(), n


def test_steps_write_the_same_files_as_host_decode(voc_tree):
    from irn_b200.step import cam_to_ir_label, make_cam, make_ins_seg_labels, make_sem_seg_labels
    root, ids, one = voc_tree
    runs = {tag: _args(root, tag, "all.txt", device_jpeg=dj) for tag, dj in (("host", False), ("exact", "exact"))}
    for a in runs.values():
        make_cam.run(a)           # mixed sizes: the 80x112 and 75x100 buckets ride on larger canvases
        make_sem_seg_labels.run(a)
        make_ins_seg_labels.run(a)
        cam_to_ir_label.run(a)
    h, e = runs["host"], runs["exact"]
    _same_npy(h.cam_out_dir, e.cam_out_dir, ids)
    _same_png(h.sem_seg_out_dir, e.sem_seg_out_dir, ids)
    _same_npy(h.ins_seg_out_dir, e.ins_seg_out_dir, ids)
    _same_png(h.ir_label_out_dir, e.ir_label_out_dir, ids)
    # a one-size list (full buckets, the one-size CAM stage), and the one-image loop of cam_to_ir_label (reads e's CAMs)
    one_runs = [_args(root, tag + "_one", "one.txt", device_jpeg=dj) for tag, dj in (("host", False), ("exact", "exact"))]
    for a in one_runs:
        make_cam.run(a)
    _same_npy(one_runs[0].cam_out_dir, one_runs[1].cam_out_dir, one)
    loop = _args(root, "exact_loop", "all.txt", device_jpeg="exact", step_batch=1, cam_out_dir=e.cam_out_dir)
    cam_to_ir_label.run(loop)
    _same_png(h.ir_label_out_dir, loop.ir_label_out_dir, ids)
