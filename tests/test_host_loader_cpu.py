"""Host-side loader logic of the steps (C1 data path), on the CPU: item formats of the datasets in both modes, the
batch-size-1 collation the steps rely on, the stride partition of the shards, run_sample's flag table."""
import os
import types

import numpy as np
import torch
from PIL import Image

from irn_b200.misc import torchutils
from irn_b200.step import _common
from irn_b200.voc12 import dataloader as dl
from irn_b200 import synth


def _voc_tree(tmp_path, sizes):
    root = tmp_path / "voc"
    os.makedirs(root / "JPEGImages")
    ids, labels = [], {}
    for i, (H, W) in enumerate(sizes):
        name = "2007_%06d" % (32 + i)
        Image.fromarray(synth.image(i, H, W)).save(root / "JPEGImages" / (name + ".jpg"), format="PNG")   # lossless pixels
        ids.append(name)
        labels[int(name.replace("_", ""))] = synth.label(i)
    (root / "list.txt").write_text("\n".join(ids) + "\n")
    dl._cls_labels["voc12/cls_labels.npy"] = labels
    return root, ids


def test_msf_dataset_item_formats(tmp_path):
    sizes = [(37, 50), (40, 33)]
    root, ids = _voc_tree(tmp_path, sizes)
    scales = (1.0, 0.5, 1.5)
    full = dl.VOC12ClassificationDatasetMSF(str(root / "list.txt"), str(root), scales=scales)
    dec = dl.VOC12ClassificationDatasetMSF(str(root / "list.txt"), str(root), scales=scales, decode_only=True)
    assert len(full) == len(dec) == 2
    for i, (H, W) in enumerate(sizes):
        a, b = full[i], dec[i]
        assert a["name"] == b["name"] == ids[i] and a["size"] == b["size"] == (H, W)
        assert torch.equal(a["label"], b["label"]) and a["label"].shape == (20,)
        assert "img_u8" not in a and "img" not in b
        assert b["img_u8"].dtype == np.uint8 and b["img_u8"].shape == (H, W, 3) and b["img_u8"].flags.writeable
        assert np.array_equal(b["img_u8"], synth.image(i, H, W))
        assert [x.shape for x in a["img"]] == [(2, 3, H, W), (2, 3, round(H * 0.5), round(W * 0.5)), (2, 3, round(H * 1.5), round(W * 1.5))]
        assert np.array_equal(a["img"][0][1], a["img"][0][0][..., ::-1])          # second entry = W-flip (voc12/dataloader.py:199)
    one = dl.VOC12ClassificationDatasetMSF(str(root / "list.txt"), str(root), scales=(1.0,))[0]["img"]
    assert isinstance(one, np.ndarray) and one.shape == (2, 3, 37, 50)            # single scale: no list (voc12/dataloader.py:200-201)


def test_collate_one_and_shards(tmp_path):
    ds = dl.SyntheticMSF(5, size=(32, 48), scales=(1.0, 0.5), decode_only=True)
    pack = _common.collate_one([ds[3]])
    assert pack["size"] == (32, 48) and all(isinstance(v, int) for v in pack["size"])
    assert pack["img_u8"].shape == (1, 32, 48, 3) and pack["img_u8"].dtype == torch.uint8
    assert pack["label"].shape == (1, 20) and pack["name"] == ["2007_000003"]
    shards = torchutils.split_dataset(ds, 2)
    assert [len(s) for s in shards] == [3, 2]
    assert [s[0]["name"] for s in shards] == ["2007_000000", "2007_000001"]     # rank r takes r, r+n, ... (misc/torchutils.py:66-68)
    assert getattr(getattr(shards[0], "dataset", shards[0]), "scales") == (1.0, 0.5)   # what work_loop hands to attach_pyramid
    args = types.SimpleNamespace(synthetic=4, voc12_root="")
    assert _common.device_pyramid(args) is True
    assert _common.make_dataset(args, "/nonexistent/list.txt", (1.0,)).decode_only is True
    args.device_pyramid = False
    assert _common.make_dataset(args, "/nonexistent/list.txt", (1.0,)).decode_only is False
    assert _common.attach_pyramid({"img": "kept"}, (1.0,)) == {"img": "kept"}     # host-pyramid items pass through untouched


def test_run_sample_flag_table():
    import run_sample
    names = [f[0] for f in run_sample.FLAGS]
    assert len(names) == len(set(names)) and {"device_pyramid", "synthetic", "cam_scales", "beta", "exp_times"} <= set(names)
    assert run_sample._bool("False") is False and run_sample._bool("true") is True
    assert run_sample._scales("1.0,0.5") == (1.0, 0.5)


def test_spawn_arguments_pickle():
    """What `torch.multiprocessing.spawn(_work, args=(model, shards, args))` has to pickle when there is more than one GPU
    (step/make_cam.py:74): the model (parameter holder, no device plan yet), the strided shards of both dataset kinds,
    the argument namespace -- and the shards must still yield items after the round trip."""
    import pickle
    from irn_b200.cam import CAM
    from irn_b200.irn import EdgeDisplacement
    args = types.SimpleNamespace(synthetic=6, voc12_root="", num_workers=0, cam_scales=(1.0, 0.5))
    shards = torchutils.split_dataset(_common.make_dataset(args, "unused", args.cam_scales), 2)
    for model in (CAM(), EdgeDisplacement()):
        model.load_state_dict(model.state_dict())
        blob = pickle.dumps((model, shards, args))
        m2, s2, a2 = pickle.loads(blob)
        assert len(m2.state_dict()) == len(model.state_dict()) and m2._plan is None
        assert [len(s) for s in s2] == [3, 3] and s2[1][0]["name"] == "2007_000001"
        assert s2[0][1]["img_u8"].shape == (512, 512, 3) and a2.synthetic == 6


def test_synthetic_names_are_the_same_for_every_step(tmp_path):
    """--synthetic: make_cam (reads --train_list in the reference) and the label steps (--infer_list) must see the same ids,
    whatever list files happen to exist in the working directory; --synthetic_list names them explicitly."""
    (tmp_path / "train_aug.txt").write_text("2007_000032\n2007_000039\n")
    (tmp_path / "train.txt").write_text("2008_000001\n2008_000002\n")
    args = types.SimpleNamespace(synthetic=2, voc12_root="")
    a = _common.make_dataset(args, str(tmp_path / "train_aug.txt"), (1.0,))
    b = _common.make_dataset(args, str(tmp_path / "train.txt"), (1.0,))
    assert [a[i]["name"] for i in range(2)] == [b[i]["name"] for i in range(2)] == ["2007_000000", "2007_000001"]
    args.synthetic_list = str(tmp_path / "train_aug.txt")
    c = _common.make_dataset(args, str(tmp_path / "train.txt"), (1.0,))
    assert [c[i]["name"] for i in range(2)] == ["2007_000032", "2007_000039"]
    assert _common.step_batch(args) == _common.DEFAULT_STEP_BATCH and _common.step_batch(types.SimpleNamespace(step_batch=1)) == 1


def test_loader_attaches_stored_cams(tmp_path):
    """Label steps in batched mode: the loader worker reads make_cam's .npy (keys + stride-4 CAMs, not the full-resolution maps)
    and the batch-1 collation keeps them usable (voc12.dataloader.attach_cam, step/_common.load_cam_dicts)."""
    cam_dir = tmp_path / "cam"
    os.makedirs(cam_dir)
    for i in range(2):
        np.save(cam_dir / ("2007_%06d.npy" % i), {"keys": torch.tensor([3, 11]), "cam": torch.full((2, 8, 12), float(i)),
                                                    "high_res": np.zeros((2, 32, 48), np.float32)})
    ds = dl.SyntheticMSF(2, size=(32, 48), scales=(1.0,), decode_only=True, cam_dir=str(cam_dir))
    pack = _common.collate_one([ds[1]])
    assert pack["cam"].shape == (1, 2, 8, 12) and float(pack["cam"].max()) == 1.0 and pack["cam_keys"].tolist() == [[3, 11]]
    args = types.SimpleNamespace(synthetic=2, voc12_root="", step_batch=1)
    assert _common.make_dataset(args, "x", (1.0,), cam_dir=str(cam_dir)).cam_dir is None      # one-image loop: the step reads the file itself
    args.step_batch = 8
    assert _common.make_dataset(args, "x", (1.0,), cam_dir=str(cam_dir)).cam_dir == str(cam_dir)


def test_chunked_messages_with_exact_bytes_split_back_into_batch1_packs(tmp_path):
    """Batched mode ships LOADER_CHUNK items per worker message (step/_common.collate_chunk: one flat tensor for the pixels / JPEG
    bytes, one for the stored CAMs); split_chunk must give back exactly the packs of the batch-size-1 collation, in order,
    including ragged items (different image sizes, different K, a JPEG byte stream next to decoded pixels)."""
    from torch.utils.data import DataLoader
    cam_dir = tmp_path / "cam"
    os.makedirs(cam_dir)
    rng = np.random.RandomState(0)
    items = []
    for i, (h, w, k) in enumerate([(24, 32, 1), (24, 32, 3), (16, 20, 2)]):
        item = {"name": "2007_%06d" % i, "size": (h, w), "label": torch.from_numpy(rng.rand(20).astype(np.float32)),
                "cam_keys": torch.arange(k, dtype=torch.int64) + i, "cam": torch.from_numpy(rng.rand(k, h // 4, w // 4).astype(np.float32))}
        if i == 1:
            item["jpeg_exact"] = rng.randint(0, 255, 777).astype(np.uint8)
        else:
            item["img_u8"] = rng.randint(0, 255, (h, w, 3)).astype(np.uint8)
        items.append(item)
    packs = list(_common.split_chunk(_common.collate_chunk([dict(it) for it in items])))
    assert len(packs) == 3
    for it, p in zip(items, packs):
        ref = _common.collate_one([dict(it)])
        assert set(p) == set(ref)
        assert p["name"] == ref["name"] and p["size"] == ref["size"]
        for k in ("label", "cam", "cam_keys", "img_u8", "jpeg_exact"):
            if k in ref:
                assert p[k].shape == ref[k].shape and p[k].dtype == ref[k].dtype and torch.equal(p[k], ref[k]), k
    # through a real DataLoader with workers, over a stride shard: same items, same order as the batch-1 loader
    ds = dl.SyntheticMSF(11, size=(24, 32), scales=(1.0,), decode_only=True)
    shard = torchutils.split_dataset(ds, 2)[1]
    got = [p for msg in DataLoader(shard, shuffle=False, batch_size=_common.LOADER_CHUNK // 2, num_workers=2, collate_fn=_common.collate_chunk)
           for p in _common.split_chunk(msg)]
    ref = list(DataLoader(shard, shuffle=False, num_workers=0, collate_fn=_common.collate_one))
    assert [p["name"] for p in got] == [p["name"] for p in ref] == [["2007_%06d" % i] for i in (1, 3, 5, 7, 9)]
    for a, b in zip(got, ref):
        assert a["size"] == b["size"] and torch.equal(a["img_u8"], b["img_u8"]) and torch.equal(a["label"], b["label"])
