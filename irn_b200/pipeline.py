"""Batched pseudo-label pipeline: the reference's make_cam -> make_sem_seg_labels / make_ins_seg_labels chains
(step/make_cam.py:28-56, step/make_sem_seg_labels.py:28-51, step/make_ins_seg_labels.py:122-152) for a batch of
images, kept on the device end to end (the reference round-trips every image through a .npy file and one-image kernels).
Every stage also comes in a form for images of different sizes, exact to the one-size form: the CAM stage on per-sub-batch
canvases with masked padding (cam_ragged_stage), the IRNet, walk, label and instance stages on the padded crop_size canvas
(*_ragged_stage, walk_padded_stage).

    stage                      reference                                    here
    pyramids (C1)              voc12/dataloader.py:191-201                  PseudoLabelPipeline.pyramids
    multi-scale CAM (C2-C4)    step/make_cam.py:35-52                       .cam_stage, .cam_ragged_stage
    EdgeDisplacement (I1/I2)   step/make_sem_seg_labels.py:32               .irn_stage, .irn_ragged_stage
    random walk (R1-R6)        misc/indexing.py:141-167                     .walk_stage, .walk_padded_stage
    label map (S1)             step/make_sem_seg_labels.py:43-49            .label_stage, .label_ragged_stage
    instances (P1-P4)          step/make_ins_seg_labels.py:131-150          .instance_stage, .instance_ragged_stage

`irn_b200.step.*` drive these stages from the reference's `run(args)` entry points (files in, files out); `run_u8` /
`run_instances_u8` chain them in memory.
"""
import numpy as np
import torch

from . import cam_ops, indexing, instance, preprocess
from .voc12 import dataloader as voc_data

KNEE_PIXELS = 512 * 512   # the sub-batches below are sized for images up to this many pixels (PASCAL VOC's) and shrink beyond


def preprocess_batch(images_u8, scales=(1.0, 0.5, 1.5, 2.0), pin=True):
    """C1 on the host (voc12/dataloader.py:185-205): list of uint8 [H,W,3] of one size -> list over scales of
    float32 tensors [2N,3,h_s,w_s] (image, flipped image interleaved), pinned for async H2D."""
    per_scale = [[] for _ in scales]
    for img in images_u8:
        ms = voc_data.multi_scale_flip(img, scales)
        ms = ms if isinstance(ms, list) else [ms]
        for s, a in enumerate(ms):
            per_scale[s].append(a)
    out = []
    for lst in per_scale:
        t = torch.from_numpy(np.ascontiguousarray(np.concatenate(lst, 0)))
        out.append(t.pin_memory() if pin and torch.cuda.is_available() else t)
    return out


class PseudoLabelPipeline:
    def __init__(self, cam_model, irn_model, device, scales=(1.0, 0.5, 1.5, 2.0), beta=10, exp_times=8, bg_thres=0.25,
                 cam_sub_batch=8, rw_sub_batch=64):
        self.cam, self.irn, self.device = cam_model, irn_model, device
        self.scales, self.beta, self.exp_times, self.bg = tuple(scales), beta, exp_times, bg_thres
        self.cam_sub, self.rw_sub = cam_sub_batch, rw_sub_batch
        self._copy_stream = None
        self._staging = {}

    # ------------------------------------------------------------------ stages
    def _cam_sub_batch(self, scale, size):
        """Image pairs per CAM forward at `scale`: cam_sub at scale 2.0, more at smaller scales, fewer for images above 512 x 512
        pixels (MS COCO's reach 640), so that a forward's activation arena holds about cam_sub 1024 x 1024 canvases at most."""
        big = min(1.0, float(KNEE_PIXELS) / (int(size[0]) * int(size[1])))
        return max(1, int(self.cam_sub * (2.0 / scale) ** 2 * big))

    def _irn_sub_batch(self):
        """Images per IRNet forward: 4 cam_sub on the 512 x 512 canvas, fewer on a larger one (--irn_crop_size 640 for MS COCO)."""
        return max(1, int(self.cam_sub * 4 * min(1.0, float(KNEE_PIXELS) / int(self.irn.crop_size) ** 2)))

    def _upload_u8(self, images_u8, slot="u8"):
        x = images_u8
        if not x.is_cuda:
            buf = self._staging.get(slot)
            if buf is None or buf.shape != x.shape:
                buf = torch.empty(x.shape, dtype=torch.uint8, device=self.device)
                self._staging[slot] = buf
            buf.copy_(x, non_blocking=True)
            x = buf
        return x

    def pyramids(self, images_u8, scales=None):
        """C1 on the device: uint8 [N,H,W,3] (cuda, or pinned host -> copied) -> list over scales of fp32 [2N,3,h_s,w_s]
        in persistent buffers, bit-exact with the reference's PIL loader (irn_b200.preprocess)."""
        scales = self.scales if scales is None else tuple(scales)
        x = self._upload_u8(images_u8)
        N, H, W = int(x.shape[0]), int(x.shape[1]), int(x.shape[2])
        out = []
        for s in scales:
            oh, ow = (H, W) if s == 1 else preprocess.rescaled_size(H, W, s)
            key = ("pyr", float(s))
            buf = self._staging.get(key)
            if buf is None or tuple(buf.shape) != (2 * N, 3, oh, ow):
                buf = torch.empty((2 * N, 3, oh, ow), dtype=torch.float32, device=self.device)
                self._staging[key] = buf
            out.append(preprocess.resize_normalize(x, (oh, ow), out=buf))
        return out

    def cam_stage(self, xs, labels, size, want_highres=True, scales=None, ready=None, order=None):
        """C2-C4: per-scale CAM forward in sub-batches of image pairs, then merge + normalise per image
        (step/make_cam.py:35-52).  xs: list over scales of cuda [2N,3,h_s,w_s]; labels [N,C] multi-hot.
        Returns (keys: list of int64 arrays, strided: list of cuda [K_i,h4,w4], highres: list of cuda [K_i,H,W] or None)."""
        scales = self.scales if scales is None else tuple(scales)
        main = torch.cuda.current_stream(self.device)
        N = xs[0].shape[0] // 2
        cams = [None] * len(xs)
        for k in (order if order is not None else range(len(xs))):
            x, s = xs[k], scales[k]
            if ready is not None and ready[k] is not None:
                main.wait_event(ready[k])
            # sub-batch so that every forward sees about the same number of pixels (cam_sub images at scale 2.0):
            # small scales batch more images to keep all SMs busy, large scales bound the activation arena
            sub = self._cam_sub_batch(s, size)
            outs = [self.cam.forward_batch(x[2 * i:2 * min(i + sub, N)]) for i in range(0, N, sub)]
            cams[k] = outs[0] if len(outs) == 1 else torch.cat(outs, 0)
        keys, strided, highres = [], [], []
        for i in range(N):
            k, lo, hi = cam_ops.merge_cams([c[i] for c in cams], size, labels[i], want_highres=want_highres)
            keys.append(k.numpy())
            strided.append(lo)
            highres.append(hi)
        return keys, strided, (highres if want_highres else None)

    def cam_ragged_stage(self, images_u8, sizes, labels, want_highres=True, scales=None):
        """C1-C4 for images of different sizes: images_u8 one flat cuda uint8 buffer holding uint8 [H_i,W_i,3] back to back, sizes
        [(H_i, W_i)], labels [N,C].  Per scale, the sub-batches of cam_stage, each on a canvas as large as its largest image
        (preprocess.resize_normalize_ragged, CAM.forward_ragged); then merge + normalise per image on its own corner of the CAMs.
        Returns what cam_stage returns, each image's entries bit for bit those cam_stage gives for it."""
        scales = self.scales if scales is None else tuple(scales)
        sizes = [(int(h), int(w)) for h, w in sizes]
        N = len(sizes)
        offs = np.concatenate([[0], np.cumsum([3 * h * w for h, w in sizes])])
        cams = [[] for _ in range(N)]
        for s in scales:
            sub = self._cam_sub_batch(s, max(sizes, key=lambda hw: hw[0] * hw[1]))     # as cam_stage
            for i in range(0, N, sub):
                j = min(i + sub, N)
                canvas, ext = preprocess.resize_normalize_ragged(images_u8[int(offs[i]):int(offs[j])], sizes[i:j], s)
                out = self.cam.forward_ragged(canvas, ext)
                for k, (h, w) in enumerate(ext):
                    cams[i + k].append(out[k, :, :(h - 1) // 16 + 1, :(w - 1) // 16 + 1])
        keys, strided, highres = [], [], []
        for i in range(N):
            k, lo, hi = cam_ops.merge_cams(cams[i], sizes[i], labels[i], want_highres=want_highres)
            keys.append(k.numpy())
            strided.append(lo)
            highres.append(hi)
        return keys, strided, (highres if want_highres else None)

    def irn_stage(self, x1):
        """I1/I2: x1 cuda fp32 [2N,3,H,W] (scale-1.0 pyramid) -> (edge [N,h,w], dp [N,2,h,w])."""
        N = x1.shape[0] // 2
        irn_sub = self._irn_sub_batch()
        edges, dps = [], []
        for i in range(0, N, irn_sub):
            e, d = self.irn.forward_batch(x1[2 * i:2 * min(i + irn_sub, N)])
            edges.append(e[:, 0])
            dps.append(d)
        return (edges[0], dps[0]) if len(edges) == 1 else (torch.cat(edges, 0), torch.cat(dps, 0))

    def irn_ragged_stage(self, images_u8, sizes):
        """I1/I2 for images of different sizes: images_u8 one flat cuda uint8 buffer holding uint8 [H_i,W_i,3] back to back, sizes
        [(H_i, W_i)] -> (edge [N,fc,fc], dp [N,2,fc,fc]) on the crop_size canvas (EdgeDisplacement.forward_ragged)."""
        irn_sub = self._irn_sub_batch()
        offs = np.concatenate([[0], np.cumsum([3 * h * w for h, w in sizes])])
        edges, dps = [], []
        for i in range(0, len(sizes), irn_sub):
            j = min(i + irn_sub, len(sizes))
            e, d = self.irn.forward_ragged(images_u8[int(offs[i]):int(offs[j])], sizes[i:j])
            edges.append(e[:, 0])
            dps.append(d)
        return (edges[0], dps[0]) if len(edges) == 1 else (torch.cat(edges, 0), torch.cat(dps, 0))

    def walk_padded_stage(self, seeds, edges, sizes):
        """walk_stage for images of different sizes on the padded grids of irn_ragged_stage: seeds [C_i,fh_i,fw_i] are zero-padded
        to the edges' fc x fc; returns the list of walks cropped back to [C_i,fh_i,fw_i].  Exactly the walk on each image's own grid:
        the padded edge is 1.0, so every path into the pad has affinity 0, and a path between two pixels of the image stays inside it."""
        fc_h, fc_w = int(edges.shape[-2]), int(edges.shape[-1])
        padded = [torch.nn.functional.pad(s, (0, fc_w - s.shape[-1], 0, fc_h - s.shape[-2])) for s in seeds]
        rw, counts = self.walk_stage(padded, edges)
        out, o = [], 0
        for (h, w), c in zip(sizes, counts):
            fh, fw = (h - 1) // 4 + 1, (w - 1) // 4 + 1
            out.append(rw[o:o + c, :fh, :fw])
            o += c
        return out

    def label_ragged_stage(self, rws, keys, sizes, bg_thres=None):
        """S1 for images of different sizes: rws list of [C_i,fh_i,fw_i] walks -> one flat cuda uint8 buffer holding the label maps
        [H_i,W_i] back to back."""
        out = torch.empty(sum(h * w for h, w in sizes), dtype=torch.uint8, device=self.device)
        o = 0
        for rw, k, (h, w) in zip(rws, keys, sizes):
            lab = out[o:o + h * w].view(h, w)
            if rw.shape[0]:
                indexing.rw_labels(rw, k, (h, w), self.bg if bg_thres is None else bg_thres, out=lab)
            else:
                lab.zero_()
            o += h * w
        return out

    def instance_ragged_stage(self, strided, keys, edges, dps, sizes, bg_thres=None):
        """instance_stage for images of different sizes on the padded grids of irn_ragged_stage: the displacement field is cropped to
        each image's [2,fh_i,fw_i] before the centroid search, the walk runs padded (walk_padded_stage)."""
        seeds, n_inst = [], []
        for i, (h, w) in enumerate(sizes):
            dp = dps[i, :, :(h - 1) // 4 + 1, :(w - 1) // 4 + 1].contiguous()
            cen = instance.find_centroids_with_refinement(dp)
            inst_map, I = instance.cluster_centroids(cen, dp)
            n_inst.append(I)
            s = instance.separate_score_by_mask(strided[i], inst_map, I)            # [K, I, h, w]
            seeds.append(s.reshape(-1, s.shape[-2], s.shape[-1]))
        rws = self.walk_padded_stage(seeds, edges, sizes)
        return [self._detections(rw, k, I, size, bg_thres) for rw, k, I, size in zip(rws, keys, n_inst, sizes)]

    def _detections(self, rw, keys, n_inst, size, bg_thres):
        """P4 of one image (step/make_ins_seg_labels.py:137-150): its walk [K*I,h,w] -> the reference's detection dict, None
        without detections."""
        if rw.shape[0] == 0:
            return None
        _, index, scores = indexing.rw_labels(rw, None, size, self.bg if bg_thres is None else bg_thres, want_index=True, want_scores=True)
        try:
            return instance.detect_instance(scores, index, np.repeat(np.asarray(keys), n_inst), max_fragment_size=size[0] * size[1] * 0.01)
        except ValueError:
            return None

    def walk_stage(self, seeds, edges):
        """R1-R6 batched: seeds = list over images of cuda [C_i,h,w]; edges [N,h,w].  Returns (rw [sum C_i,h,w], counts).
        The fused cluster kernel takes every (image, channel) of a sub-batch in one launch."""
        N = len(seeds)
        counts = [int(s.shape[0]) for s in seeds]
        rws = []
        for i in range(0, N, self.rw_sub):
            j = min(i + self.rw_sub, N)
            offs = np.concatenate([[0], np.cumsum(counts[i:j])])
            sd = seeds[i] if j - i == 1 else torch.cat(seeds[i:j], 0)
            rws.append(indexing.random_walk_batch(sd, edges[i:j], offs, 5, self.beta, 2 ** self.exp_times))
        return (rws[0] if len(rws) == 1 else torch.cat(rws, 0)), counts

    def label_stage(self, rw, counts, keys, size, bg_thres=None):
        """S1: label maps uint8 cuda [N,H,W] (images without a class are all background, like an empty CAM dict)."""
        N = len(counts)
        out = torch.empty((N, size[0], size[1]), dtype=torch.uint8, device=self.device)
        o = 0
        for i in range(N):
            if counts[i]:
                indexing.rw_labels(rw[o:o + counts[i]], keys[i], size, self.bg if bg_thres is None else bg_thres, out=out[i])
            else:
                out[i].zero_()
            o += counts[i]
        return out

    def instance_stage(self, strided, keys, edges, dps, size, bg_thres=None, to_host=True):
        """P1-P4 for a batch (step/make_ins_seg_labels.py:131-150): per image centroids -> clusters -> per-instance
        seeds; ONE batched walk over all K_i x I_i channels; per image x4 up / max / bg / argmax and detections.
        Returns a list of the reference's dicts {'score','mask','class'} (numpy), None for an image without detections
        (the reference raises on np.stack([]) there)."""
        N = len(strided)
        seeds, n_inst = [], []
        for i in range(N):
            cen = instance.find_centroids_with_refinement(dps[i])
            inst_map, I = instance.cluster_centroids(cen, dps[i])
            n_inst.append(I)
            s = instance.separate_score_by_mask(strided[i], inst_map, I)            # [K, I, h, w]
            seeds.append(s.reshape(-1, s.shape[-2], s.shape[-1]))
        rw, counts = self.walk_stage(seeds, edges)
        out, o = [], 0
        for i in range(N):
            out.append(self._detections(rw[o:o + counts[i]], keys[i], n_inst[i], size, bg_thres))
            o += counts[i]
        return out

    # ------------------------------------------------------------------ whole chains
    @torch.no_grad()
    def run_u8(self, images_u8, labels, want_highres=True):
        """make_cam -> make_sem_seg_labels starting from decoded images: uint8 [N,H,W,3], cuda or (pinned) host.  The
        per-scale bicubic rescale, normalisation and flip stack of the reference's loader run on the device, bit-exact,
        so a step uploads 0.79 MB per 512x512 image instead of 47 MB of fp32 pyramids."""
        if 1.0 not in self.scales:
            raise ValueError("the IRNet pass uses the scale-1.0 input (step/make_sem_seg_labels.py:64-66)")
        H, W = int(images_u8.shape[1]), int(images_u8.shape[2])
        return self.run(self.pyramids(images_u8), labels, (H, W), want_highres)

    @torch.no_grad()
    def run(self, inputs, labels, size, want_highres=True):
        """inputs: list over scales of [2N,3,h_s,w_s] fp32 (cuda, or pinned host -> copied here);
        labels: [N,C] multi-hot; size=(H,W).  Returns dict with 'labels' uint8 cuda [N,H,W], 'keys' list,
        'cams' list of cuda [K_i,h4,w4] and 'high_res' list (or None)."""
        dev = self.device
        # host inputs: copy on a side stream, one event per scale, so the forward of scale k overlaps the H2D of scale k+1..
        main = torch.cuda.current_stream(dev)
        if any(not x.is_cuda for x in inputs):
            if self._copy_stream is None:
                self._copy_stream = torch.cuda.Stream(device=dev)
            self._copy_stream.wait_stream(main)          # buffers freed on the main stream may be recycled for the copies
        order = sorted(range(len(inputs)), key=lambda k: inputs[k].numel())     # smallest scale first: least exposed copy
        xs, ready = [None] * len(inputs), [None] * len(inputs)
        for k in order:
            x = inputs[k]
            if x.is_cuda:
                xs[k] = x
            else:
                # persistent device staging buffers (no allocator traffic across streams); the wait_stream above guarantees the
                # previous step has finished reading them
                buf = self._staging.get(k)
                if buf is None or buf.shape != x.shape:
                    buf = torch.empty(x.shape, dtype=torch.float32, device=dev)
                    self._staging[k] = buf
                with torch.cuda.stream(self._copy_stream):
                    buf.copy_(x, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(self._copy_stream)
                xs[k] = buf
                ready[k] = ev
        keys, strided, highres = self.cam_stage(xs, labels, size, want_highres, ready=ready, order=order)
        edges, dps = self.irn_stage(xs[self.scales.index(1.0)])
        rw, counts = self.walk_stage(strided, edges)
        out = self.label_stage(rw, counts, keys, size)
        return {"labels": out, "keys": keys, "cams": strided, "high_res": highres, "edge": edges, "dp": dps}

    @torch.no_grad()
    def run_instances_u8(self, images_u8, keys, strided):
        """make_ins_seg_labels for a batch (step/make_ins_seg_labels.py:122-152): decoded uint8 images + the stored CAMs
        of make_cam (`keys`, `strided` as returned by cam_stage / read from the .npy files) -> list of detection dicts."""
        H, W = int(images_u8.shape[1]), int(images_u8.shape[2])
        x1 = self.pyramids(images_u8, (1.0,))[0]
        edges, dps = self.irn_stage(x1)
        return self.instance_stage(strided, keys, edges, dps, (H, W))
