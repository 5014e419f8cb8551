"""Drop-in for the reference's ``step/cam_to_ir_label.py``: the confident foreground / background label maps of the stored CAMs,
each refined by the fully connected CRF, combined into the IRNet training label (0 = background, 255 = unsure, else class + 1)
and written as ``ir_label_out_dir/<name>.png`` (step/cam_to_ir_label.py:12-43).  The CRF runs on the GPU (irn_b200.crf); both CRFs
of an image share its two lattices."""
import os

import numpy as np
import torch
from PIL import Image

from .. import crf
from ..voc12 import dataloader as voc_data
from . import _common


def _write(labels, path):
    # compress_level 1: the same pixels as the reference's imageio PNG, a fraction of zlib's default time
    Image.fromarray(labels).save(path, compress_level=1)


def ir_label_one_image(model, pack, args):
    """step/cam_to_ir_label.py:19-41 for one image (the reference's loop; --step_batch 1)."""
    name = voc_data.decode_int_filename(pack["name"][0])
    cam_dict = np.load(os.path.join(args.cam_out_dir, name + ".npy"), allow_pickle=True).item()
    img = pack["img_u8"].cuda(non_blocking=True)
    conf = crf.ir_labels(img, [cam_dict["high_res"]], [np.asarray(cam_dict["keys"])], args.conf_fg_thres, args.conf_bg_thres)
    _write(conf[0].cpu().numpy(), os.path.join(args.ir_label_out_dir, name + ".png"))


def _save(ctx, names, conf, out_dir):
    (lab,) = ctx.writer.to_host([conf])
    lab = lab.numpy()
    for i, name in enumerate(names):
        ctx.writer.submit_file(_write, lab[i], os.path.join(out_dir, name + ".png"))


def ir_label_batch(ctx, packs):
    """The same body for a bucket of equally-sized images: one batched CRF call for all of them."""
    args = ctx.args
    names = [voc_data.decode_int_filename(p["name"][0]) for p in packs]
    with ctx.phase("cam dicts"):
        keys, high = _common.load_cam_dicts(ctx, packs, names, args.cam_out_dir, field="high_res")
    with ctx.phase("stack + upload images"):
        x = ctx.stack_images(packs)
    with ctx.phase("crf"):
        conf = crf.ir_labels(x, [torch.as_tensor(h) for h in high], keys, args.conf_fg_thres, args.conf_bg_thres)
    with ctx.phase("hand to writer"):
        ctx.writer.submit(_save, ctx, names, conf, args.ir_label_out_dir)


def _work(process_id, infer_dataset, args):
    _common.work_loop(process_id, None, infer_dataset, args, ir_label_one_image, ir_label_batch)


def _work_spawn(process_id, model, dataset, args):
    _work(process_id, dataset, args)


def run(args):
    _common.run_step(args, _work_spawn, None, None, None, None, args.train_list, (1.0,), cam_dir=args.cam_out_dir, cam_field="high_res")
