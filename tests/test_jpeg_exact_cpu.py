"""The exact JPEG decoder's host side: its oracle (oracle/jpeg.py) against PIL bit for bit, the header inspection that decides which
streams the device decoder takes (irn_b200.jpeg.inspect, the C ABI's irn_jpeg_exact_inspect), --device_jpeg parsing and the
loader's routing of file bytes vs host-decoded pixels."""
import io
import os
import sys
import types

import numpy as np
import pytest
from PIL import Image, features

from conftest import golden_path
from irn_b200 import _lib, jpeg, synth
from oracle import jpeg as oracle_jpeg

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_jpeg_golden  # noqa: E402


@pytest.fixture(scope="module")
def fixture():
    g = np.load(golden_path("jpeg_exact.npz"))
    return g, [(str(g["name%d" % i]), g["jpeg%d" % i].tobytes(), g["pixels%d" % i]) for i in range(int(g["n"]))]


def test_oracle_equals_pil_on_every_fixture_case(fixture):
    _, cases = fixture
    for name, data, pixels in cases:
        got = oracle_jpeg.decode(data)
        assert got.dtype == np.uint8 and np.array_equal(got, pixels), name


def test_oracle_equals_pil_live(fixture):
    """The fixture's cases re-encoded and decoded by the installed PIL (same libjpeg-turbo as the fixture only), plus fresh
    synthetic and saturated images at the step sizes."""
    g, _ = fixture
    if (features.version("libjpeg_turbo") or "") != str(g["libjpeg_turbo"]):
        pytest.skip("installed libjpeg-turbo %s differs from the fixture's %s" % (features.version("libjpeg_turbo"), g["libjpeg_turbo"]))
    cases = make_jpeg_golden.cases()[::7]
    for q, ss in ((90, 2), (60, 1), (100, 0)):
        img = make_jpeg_golden.pattern("synth", 75 + ss, 101 - ss, q)
        cases.append(("live synth q%d ss%d" % (q, ss), make_jpeg_golden.encode(img, quality=q, subsampling=ss)))
        img = make_jpeg_golden.pattern("saturated", 33 + ss, 47 - ss, q)
        cases.append(("live saturated q%d ss%d" % (q, ss), make_jpeg_golden.encode(img, quality=q, subsampling=ss, optimize=True)))
    for name, data in cases:
        assert np.array_equal(oracle_jpeg.decode(data), np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))), name


def test_inspect_agrees_with_the_oracle(fixture):
    _, cases = fixture
    for name, data, pixels in cases:
        info = jpeg.inspect(data)
        assert info == oracle_jpeg.inspect(data), name
        assert info[:2] == pixels.shape[:2], name


def _enc(img, **kw):
    return make_jpeg_golden.encode(img, **kw)


def test_inspect_classifies_streams():
    img = synth.image(3, 40, 56)
    assert jpeg.inspect(_enc(img, quality=90, subsampling=2)) == (40, 56, 3, 2, 2, 0)
    assert jpeg.inspect(_enc(img, quality=90, subsampling=1, optimize=True)) == (40, 56, 3, 2, 1, 0)
    assert jpeg.inspect(_enc(img, quality=90, subsampling=0, restart_marker_blocks=4)) == (40, 56, 3, 1, 1, 4)
    assert jpeg.inspect(_enc(img[..., 0].copy(), quality=90)) == (40, 56, 1, 1, 1, 0)
    unsupported = [_enc(img, quality=90, progressive=True)]
    b = io.BytesIO()
    Image.fromarray(img).convert("CMYK").save(b, format="JPEG", quality=90)
    unsupported.append(b.getvalue())
    for data in unsupported:
        with pytest.raises(jpeg.UnsupportedJpeg):
            jpeg.inspect(data)
        with pytest.raises(oracle_jpeg.JpegUnsupported):
            oracle_jpeg.inspect(data)
    good = _enc(img, quality=90)
    sos = good.index(b"\xff\xda")
    bad = [good[:1], good[:2], good[:20], good[:sos], good[:sos + 6], good[:len(good) // 2], b"\x89PNG\r\n\x1a\n" + good[8:]]
    for data in bad:
        with pytest.raises(_lib.IrnError) as e:
            jpeg.inspect(data)
        assert not isinstance(e.value, jpeg.UnsupportedJpeg)
        with pytest.raises(oracle_jpeg.JpegBadArg):
            oracle_jpeg.inspect(data)


def test_device_jpeg_flag_parses_to_a_bool():
    import run_sample
    from irn_b200.step import _common
    for v, want in (("exact", True), ("EXACT", True), ("True", True), ("False", False)):
        a = run_sample.parse(["--device_jpeg", v])
        assert a.device_jpeg is want
        assert _common.device_jpeg(a) is want
    assert run_sample.parse([]).device_jpeg is False
    assert _common.device_jpeg(types.SimpleNamespace(device_jpeg="exact", device_pyramid=True)) is True
    assert _common.device_jpeg(types.SimpleNamespace(device_jpeg="exact", device_pyramid=False)) is False


def test_loader_routes_exact_bytes_and_host_pixels(tmp_path):
    """--device_jpeg: the worker ships the bytes of a file the exact decoder takes and decodes the others (PNG stand-in,
    progressive) on the host; the chunk message carries both kinds and splits back into the same packs."""
    from irn_b200.step import _common
    from irn_b200.voc12 import dataloader
    root = tmp_path / "voc"
    os.makedirs(root / "JPEGImages")
    ids = ["2007_%06d" % (900 + i) for i in range(4)]
    imgs = [synth.image(70 + i, 24 + 8 * i, 40) for i in range(4)]
    Image.fromarray(imgs[0]).save(root / "JPEGImages" / (ids[0] + ".jpg"), quality=90)
    Image.fromarray(imgs[1]).save(root / "JPEGImages" / (ids[1] + ".jpg"), format="PNG")
    Image.fromarray(imgs[2]).save(root / "JPEGImages" / (ids[2] + ".jpg"), quality=90, progressive=True)
    Image.fromarray(imgs[3][..., 0]).save(root / "JPEGImages" / (ids[3] + ".jpg"), quality=90)
    (root / "list.txt").write_text("\n".join(ids) + "\n")
    dataloader._cls_labels["voc12/cls_labels.npy"] = {int(n.replace("_", "")): synth.label(i, 2) for i, n in enumerate(ids)}
    args = types.SimpleNamespace(voc12_root=str(root), device_jpeg="exact", device_pyramid=True, step_batch=4, synthetic=0)
    ds = _common.make_dataset(args, str(root / "list.txt"), (1.0,))
    items = [ds[i] for i in range(4)]
    assert ["jpeg_exact" in it for it in items] == [True, False, False, True]
    for i in (1, 2):
        want = np.asarray(Image.open(root / "JPEGImages" / (ids[i] + ".jpg")).convert("RGB"))
        assert np.array_equal(items[i]["img_u8"], want)
    for i in (0, 3):
        assert items[i]["jpeg_exact"].tobytes() == (root / "JPEGImages" / (ids[i] + ".jpg")).read_bytes()
        assert items[i]["size"] == imgs[i].shape[:2]
    packs = list(_common.split_chunk(_common.collate_chunk(items)))
    for it, p in zip(items, packs):
        k = "jpeg_exact" if "jpeg_exact" in it else "img_u8"
        assert np.array_equal(p[k].numpy().reshape(-1), np.asarray(it[k]).reshape(-1))
    # exact bytes and host pixels of one size share a bucket
    host = {"size": (24, 40), "img_u8": packs[1]["img_u8"]}
    assert _common.size_key(packs[0]) == _common.size_key({"size": packs[0]["size"], "img_u8": host["img_u8"][:, :24]})
    one = _common.collate_one([dict(items[0])])
    assert "jpeg_exact" in one and one["size"] == (24, 40)
    # the raw-image steps (cam_to_ir_label) ship bytes too; --device_jpeg True is the exact decoder
    raw = _common.make_dataset(args, str(root / "list.txt"), (1.0,), raw_images=True)
    assert "jpeg_exact" in raw[0]
    on = _common.make_dataset(types.SimpleNamespace(**dict(vars(args), device_jpeg=True)), str(root / "list.txt"), (1.0,))
    assert "jpeg_exact" in on[0] and "img_u8" not in on[0]
