"""Drop-in for the reference's ``step/make_ins_seg_labels.py`` (step/make_ins_seg_labels.py:108-171): displacement
field -> centroids -> instance clusters, per-instance CAM seeds through the random walk, argmax, per-segment
detections saved as ``.npy`` ({'score','mask','class'})."""
import os

import numpy as np

from .. import indexing, instance
from . import _common


def ins_seg_one_image(model, pack, args):
    name, size = pack["name"][0], pack["size"]
    edge, dp = model(pack["img"][0].cuda(non_blocking=True))
    stored = np.load(os.path.join(args.cam_out_dir, name + ".npy"), allow_pickle=True).item()
    keys = np.asarray(stored["keys"])
    centroids = instance.find_centroids_with_refinement(dp)
    inst_map, n_inst = instance.cluster_centroids(centroids, dp)
    seeds = instance.separate_score_by_mask(stored["cam"].cuda(), inst_map, n_inst)            # [K, I, h, w]
    walk = indexing.propagate_to_edge(seeds, edge, beta=float(args.beta), exp_times=int(args.exp_times), radius=5)
    _, index, scores = indexing.rw_labels(walk, None, size, float(args.ins_seg_bg_thres), want_index=True, want_scores=True)
    detected = instance.detect_instance(scores, index, np.repeat(keys, n_inst), max_fragment_size=size[0] * size[1] * 0.01)
    np.save(os.path.join(args.ins_seg_out_dir, name + ".npy"), detected)


def ins_seg_batch(ctx, packs):
    """step/make_ins_seg_labels.py:122-152 for a batch of images of any sizes: one IRNet forward on the padded crop_size canvas, one
    batched walk over every (class, instance) channel of the batch on the padded feature grids
    (irn_b200.pipeline.instance_ragged_stage)."""
    args = ctx.args
    names = [p["name"][0] for p in packs]
    keys, cams = _common.load_cam_dicts(ctx, packs, names, args.cam_out_dir)
    x, sizes = ctx.pack_images(packs)
    edges, dps = ctx.pipe.irn_ragged_stage(x, sizes)
    strided = _common.to_device_list(ctx, cams)
    dets = ctx.pipe.instance_ragged_stage(strided, keys, edges, dps, sizes, float(args.ins_seg_bg_thres))
    ctx.check_decoded()     # the detections are on the host: the stream has passed the batch's JPEG decode
    for name, det in zip(names, dets):
        if det is None:     # the reference's np.stack([]) raises for an image without any detection
            raise ValueError("need at least one array to stack (no instance detected in %s)" % name)
        ctx.writer.submit_host(np.save, os.path.join(args.ins_seg_out_dir, name + ".npy"), det)


def _work(process_id, model, dataset, args):
    _common.work_loop(process_id, model, dataset, args, ins_seg_one_image, ins_seg_batch, ragged=True)


def run(args):
    _common.run_step(args, _work, args.irn_network, "EdgeDisplacement", args.irn_weights_name, False, args.infer_list, (1.0,),
                     cam_dir=args.cam_out_dir, model_kwargs={"crop_size": int(getattr(args, "irn_crop_size", 512))})
