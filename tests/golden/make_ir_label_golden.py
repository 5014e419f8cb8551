"""Generate tests/golden/ir_label.npz: the UNMODIFIED reference's step/cam_to_ir_label.py `_work` loop, with `pydensecrf` (not
installable here) provided by modules whose arithmetic is the oracle's (oracle/crf.py).  So the fixture pins the step's glue --
key padding, the two thresholds, the argmax, keys[pred], the 0 / class / 255 combination, the PNG -- to the reference, and the CRF
to the oracle.  Parity with pydensecrf itself is not pinned (DESIGN.md section 2).

Needs the reference checkout (oracle/refshim.py):   python tests/golden/make_ir_label_golden.py
Nothing at test time reads the reference.

Cases: the three images of steps.npz with their recorded high_res / keys, and seeded synthetic ones (irn_b200.synth: image(seed),
cam_planes_u8(K, H, W, seed) / 255 as the stored high_res, seed-chosen keys).  The inputs are not stored again: per case i the
fixture holds `name{i}`, `keys{i}`, either `steps_index{i}` (the image and high_res are steps.npz's `img{j}` / `cam_high{j}`) or
`seed{i}` + `cam_sha256{i}` (the synthetic planes are regenerated from the seed; the hash makes a drift in that generator fail
loudly), then `fg_conf_cam{i}`, `bg_conf_cam{i}`, `pred_fg{i}`, `pred_bg{i}`, `png{i}` (what the reference wrote), and for the
smallest image `q_fg{i}` (the oracle's final Q of the fg CRF)."""
import hashlib
import os
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import crf as ocrf, refshim  # noqa: E402
from irn_b200 import synth  # noqa: E402

SYNTH = [  # (H, W, K, seed)
    (375, 500, 3, 11),
    (500, 375, 1, 12),
    (512, 512, 20, 13),
    (375, 500, 0, 14),
]


class _Record:
    def __init__(self):
        self.labels, self.q = [], []


REC = _Record()
Q_CASE = 2          # steps.npz's 75x100 image: the one case whose final fg Q is stored


def install_pydensecrf():
    """Oracle-backed pydensecrf modules, put in place before refshim.install() (which only stubs absent names)."""
    root = types.ModuleType("pydensecrf")
    dm = types.ModuleType("pydensecrf.densecrf")
    um = types.ModuleType("pydensecrf.utils")

    class DenseCRF2D(ocrf.DenseCRF2D):
        def inference(self, t):
            q = super().inference(t)
            REC.q.append(q.reshape(self.n_labels, self.H, self.W))
            return q

    def unary_from_labels(labels, n_labels, gt_prob, zero_unsure=True):
        REC.labels.append(np.asarray(labels).copy())
        return ocrf.unary_from_labels(labels, n_labels, gt_prob, zero_unsure)
    dm.DenseCRF2D = DenseCRF2D
    um.unary_from_labels = unary_from_labels
    root.densecrf, root.utils = dm, um
    sys.modules.update({"pydensecrf": root, "pydensecrf.densecrf": dm, "pydensecrf.utils": um})


def cases():
    g = np.load(os.path.join(HERE, "steps.npz"))
    out = []
    for i, name in enumerate(g["ids"]):
        out.append({"name": str(name), "img": g["img%d" % i], "high": g["cam_high%d" % i].astype(np.float32),
                    "keys": g["cam_keys%d" % i].astype(np.int64), "steps_index": i})
    for j, (H, W, K, seed) in enumerate(SYNTH):
        rs = np.random.RandomState(seed)
        keys = np.sort(rs.choice(20, K, replace=False)).astype(np.int64)
        u8 = synth.cam_planes_u8(K, H, W, seed)
        out.append({"name": "2008_%06d" % (100 + j), "img": synth.image(seed, H, W), "seed": seed, "cam_u8": u8,
                    "high": synth.u8_to_cam(u8), "keys": keys})
    return out


def main():
    install_pydensecrf()
    refshim.install()
    os.chdir(refshim.REF)          # voc12/dataloader.py:24 loads 'voc12/cls_labels.npy' relative to cwd
    import torch
    from PIL import Image
    import step.cam_to_ir_label as ref_step

    class Items(torch.utils.data.Dataset):     # the items VOC12ImageDataset(img_normal=None, to_torch=False) yields
        def __init__(self, cs):
            self.cs = cs

        def __len__(self):
            return len(self.cs)

        def __getitem__(self, i):
            return {"name": self.cs[i]["name"], "img": self.cs[i]["img"]}

    cs = cases()
    tmp = tempfile.mkdtemp(prefix="irn_ir_label_")
    try:
        args = types.SimpleNamespace(num_workers=0, cam_out_dir=os.path.join(tmp, "cam"), ir_label_out_dir=os.path.join(tmp, "ir"),
                                     conf_fg_thres=0.30, conf_bg_thres=0.05)
        os.makedirs(args.cam_out_dir)
        os.makedirs(args.ir_label_out_dir)
        for c in cs:
            np.save(os.path.join(args.cam_out_dir, c["name"] + ".npy"), {"keys": torch.from_numpy(c["keys"]), "high_res": c["high"]})
        # process_id 1 of 2: the reference's progress line (`iter % (len(databin) // 20)`) divides by zero below 20 images
        ref_step._work(1, [None, Items(cs)], args)
        assert len(REC.q) == 2 * len(cs), len(REC.q)
        out = {"conf_fg_thres": np.float32(0.30), "conf_bg_thres": np.float32(0.05)}
        for i, c in enumerate(cs):
            out["name%d" % i] = np.array(c["name"])
            if "seed" in c:
                out["seed%d" % i] = np.int64(c["seed"])
                out["cam_sha256%d" % i] = np.array(hashlib.sha256(np.ascontiguousarray(c["cam_u8"]).tobytes()).hexdigest())
            else:
                out["steps_index%d" % i] = np.int64(c["steps_index"])
            out["keys%d" % i] = c["keys"]
            out["fg_conf_cam%d" % i] = REC.labels[2 * i].astype(np.uint8)
            out["bg_conf_cam%d" % i] = REC.labels[2 * i + 1].astype(np.uint8)
            qf, qb = REC.q[2 * i], REC.q[2 * i + 1]
            out["pred_fg%d" % i] = np.argmax(qf, 0).astype(np.uint8)
            out["pred_bg%d" % i] = np.argmax(qb, 0).astype(np.uint8)
            if i == Q_CASE:
                out["q_fg%d" % i] = qf.astype(np.float32)
            out["png%d" % i] = np.asarray(Image.open(os.path.join(args.ir_label_out_dir, c["name"] + ".png")))
            print("ir_label", c["name"], c["img"].shape, "K=%d" % len(c["keys"]), np.unique(out["png%d" % i]))
        out["n"] = np.int64(len(cs))
        np.savez_compressed(os.path.join(HERE, "ir_label.npz"), **out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
