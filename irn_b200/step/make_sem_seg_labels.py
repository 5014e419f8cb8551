"""Drop-in for the reference's ``step/make_sem_seg_labels.py``: IRNet edge map, random walk of the stored CAMs,
x4 upsample / background threshold / argmax, uint8 PNG per image (step/make_sem_seg_labels.py:28-51)."""
import os

import numpy as np
from PIL import Image

from .. import indexing
from ..voc12 import dataloader as voc_data
from . import _common


def sem_seg_one_image(model, pack, args):
    name = voc_data.decode_int_filename(pack["name"][0])
    edge, _ = model(pack["img"][0].cuda(non_blocking=True))
    stored = np.load(os.path.join(args.cam_out_dir, name + ".npy"), allow_pickle=True).item()
    walk = indexing.propagate_to_edge(stored["cam"].cuda(), edge, beta=float(args.beta), exp_times=int(args.exp_times), radius=5)
    labels, _, _ = indexing.rw_labels(walk, np.asarray(stored["keys"]), pack["size"], float(args.sem_seg_bg_thres))
    Image.fromarray(labels.cpu().numpy()).save(os.path.join(args.sem_seg_out_dir, name + ".png"))


def _save(ctx, names, labels, sizes, out_dir):
    (lab,) = ctx.writer.to_host([labels])
    lab = lab.numpy()
    o = 0
    for name, (h, w) in zip(names, sizes):
        # compress_level 1: same pixels in the file, a quarter of zlib's time on busy label maps (the default 6 made PNG encoding
        # the pacer of the whole step: 21 ms per 512x512 map against ~1 ms of GPU time)
        ctx.writer.submit_file(lambda a, p: Image.fromarray(a).save(p, compress_level=1), lab[o:o + h * w].reshape(h, w),
                               os.path.join(out_dir, name + ".png"))
        o += h * w


def sem_seg_batch(ctx, packs):
    """step/make_sem_seg_labels.py:28-51 for a batch of images of any sizes: one IRNet forward on the padded crop_size canvas, one
    batched walk on the padded feature grids, each image's walk cropped back to its own grid for the label map."""
    args = ctx.args
    names = [voc_data.decode_int_filename(p["name"][0]) for p in packs]
    with ctx.phase("cam dicts"):
        keys, cams = _common.load_cam_dicts(ctx, packs, names, args.cam_out_dir)
    with ctx.phase("stack + upload images"):
        x, sizes = ctx.pack_images(packs)
    with ctx.phase("irn forward (issue)"):
        edges, _ = ctx.pipe.irn_ragged_stage(x, sizes)
    with ctx.phase("upload cams"):
        seeds = _common.to_device_list(ctx, cams)
    with ctx.phase("walk (issue)"):
        rws = ctx.pipe.walk_padded_stage(seeds, edges, sizes)
    with ctx.phase("labels (issue)"):
        labels = ctx.pipe.label_ragged_stage(rws, keys, sizes, float(args.sem_seg_bg_thres))
    with ctx.phase("hand to writer"):
        ctx.writer.submit(_save, ctx, names, labels, sizes, args.sem_seg_out_dir)


def _work(process_id, model, dataset, args):
    _common.work_loop(process_id, model, dataset, args, sem_seg_one_image, sem_seg_batch, ragged=True)


def run(args):
    _common.run_step(args, _work, args.irn_network, "EdgeDisplacement", args.irn_weights_name, False, args.infer_list, (1.0,), opening="[",
                     cam_dir=args.cam_out_dir, model_kwargs={"crop_size": int(getattr(args, "irn_crop_size", 512))})
