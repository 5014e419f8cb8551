"""Drop-in for the reference's ``step/make_cam.py``: same ``run(args)`` namespace and the same ``.npy`` output --
a pickled ``{"keys": LongTensor[K], "cam": FloatTensor[K,h/4,w/4], "high_res": ndarray[K,H,W]}`` per image
(step/make_cam.py:55-56) -- with the arithmetic in libirn_b200."""
import os

import numpy as np
import torch

from .. import cam_ops
from . import _common


def cam_one_image(model, pack, args):
    """step/make_cam.py:28-56: CAM forward per scale, merge + normalise, save."""
    per_scale = [model(x[0].cuda(non_blocking=True)) for x in pack["img"]]
    keys, strided, highres = cam_ops.merge_cams(per_scale, pack["size"], pack["label"][0])
    np.save(os.path.join(args.cam_out_dir, pack["name"][0] + ".npy"),
            {"keys": keys, "cam": strided.cpu(), "high_res": highres.cpu().numpy()})


def _save(ctx, names, keys, strided, highres, out_dir):
    """Pool thread: one device->host copy per tensor kind for the whole batch (the images' maps flattened back to back: a batch may
    mix sizes), then one np.save per image."""
    lo, hi = ctx.writer.to_host([[t.reshape(-1) for t in strided], [t.reshape(-1) for t in highres]])
    o = oh = 0
    for name, k, s, h in zip(names, keys, strided, highres):
        # views of the batch's host buffers: pickling copies them, so the buffers live exactly as long as the last write
        ctx.writer.submit_file(np.save, os.path.join(out_dir, name + ".npy"),
                               {"keys": torch.from_numpy(k.astype(np.int64)), "cam": lo[o:o + s.numel()].view(s.shape).clone(),
                                "high_res": hi[oh:oh + h.numel()].view(h.shape).numpy()})
        o += s.numel()
        oh += h.numel()


def cam_batch(ctx, packs):
    """The same body for a batch of decoded images (irn_b200.pipeline stages C1-C4): a bucket of one size, or a bucket topped up
    with smaller images (_common.Batcher), which run on the bucket's canvas (cam_ragged_stage)."""
    args = ctx.args
    labels = torch.cat([p["label"] for p in packs], 0)
    with ctx.phase("pack + upload images"):
        flat, sizes = ctx.pack_images(packs)
    if len(set(sizes)) > 1:
        with ctx.phase("ragged pyramids + cam forward + merge (issue)"):
            keys, strided, highres = ctx.pipe.cam_ragged_stage(flat, sizes, labels, want_highres=True, scales=ctx.scales)
    else:
        with ctx.phase("pyramids + cam forward + merge (issue)"):
            xs = ctx.pipe.pyramids(flat.view((len(packs),) + sizes[0] + (3,)), ctx.scales)
            keys, strided, highres = ctx.pipe.cam_stage(xs, labels, packs[0]["size"], want_highres=True, scales=ctx.scales)
    with ctx.phase("hand to writer"):
        ctx.writer.submit(_save, ctx, [p["name"][0] for p in packs], keys, strided, highres, args.cam_out_dir)


def _work(process_id, model, dataset, args):
    _common.work_loop(process_id, model, dataset, args, cam_one_image, cam_batch, riders=True)


def run(args):
    # the reference appends '.pth' to --cam_weights_name here (step/make_cam.py:64) but not for the IRN weights
    _common.run_step(args, _work, args.cam_network, "CAM", args.cam_weights_name + ".pth", True, args.train_list, args.cam_scales)
