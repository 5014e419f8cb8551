"""Shared plumbing of the three label-generation steps.

The reference repeats the same skeleton in step/make_cam.py, step/make_sem_seg_labels.py and
step/make_ins_seg_labels.py: build the model class named on the command line, load its checkpoint, split the
image list over the visible GPUs with the stride partition, spawn one worker per GPU, loop over a batch-size-1
DataLoader.  Here that skeleton exists once; each step module supplies its per-image function (the reference's loop
body, one image at a time) and its per-batch function (the same arithmetic for a batch of images through irn_b200.pipeline, used
whenever the loader hands over decoded uint8 images: --device_pyramid, the default).

Batched mode keeps the reference's observable behaviour: same files, same names, same formats; only the order in which
files appear changes, and file writes overlap the GPU work of the next batch on a small thread pool.  make_sem_seg_labels and
make_ins_seg_labels batch images of any sizes (IRNet pads every image to crop_size anyway, and the walk on the padded grid is the
walk on the image's own grid), and so does cam_to_ir_label (the CRF builds each image's lattices at its own size within one ragged
call): a batch is every --step_batch consecutive images.  make_cam works at each image's own size: its images are bucketed by size,
a bucket is flushed when it holds --step_batch images, when the pending buckets together hold more than PENDING_BOUND x
--step_batch images (the largest goes), or at the end (Batcher), and a bucket flushed before it is full is topped up with smaller
images of other sizes, which its CAM forward runs on the bucket's canvas with the padding masked, exactly as at their own size.
"""
import contextlib
import importlib
import os
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from torch.utils.data import DataLoader
from torch.utils.data._utils.collate import default_collate

from .. import preprocess
from ..misc import torchutils
from ..voc12 import dataloader as voc_data

DEFAULT_STEP_BATCH = 32


def collate_one(batch):
    """batch_size=1 collation like the reference's DataLoader, except that `size` stays a pair of python ints
    (torch's default collate makes it [tensor([H]), tensor([W])], which modern numpy can no longer use as a slice
    bound, step/make_sem_seg_labels.py:29,43)."""
    stream = batch[0].pop("jpeg_exact", None) if isinstance(batch[0], dict) else None
    out = default_collate(batch)
    if stream is not None:
        out["jpeg_exact"] = torch.from_numpy(stream)        # variable-length byte stream: no batch dimension
    out["size"] = (int(batch[0]["size"][0]), int(batch[0]["size"][1]))
    return out


LOADER_CHUNK = 8


def collate_chunk(batch):
    """Several consecutive items as ONE message from a loader worker: the decoded images (or JPEG byte streams) in one flat uint8
    tensor, the stored CAMs in one flat fp32 tensor.  A DataLoader hands every tensor of every item to the main process through its
    own file-descriptor exchange (~0.5 ms each): with batch_size=1 and five tensors per item that alone caps the label steps at a
    few hundred images/s, whatever the number of workers.  `split_chunk` turns the
    message back into batch_size=1 packs (views, no copies)."""
    out = {"names": [b["name"] for b in batch], "sizes": [(int(b["size"][0]), int(b["size"][1])) for b in batch],
           "label": torch.stack([torch.as_tensor(b["label"]) for b in batch])}
    kinds, shapes, parts = [], [], []
    for b in batch:
        k = "jpeg_exact" if "jpeg_exact" in b else "img_u8"
        a = np.ascontiguousarray(b[k])
        kinds.append(k)
        shapes.append(tuple(a.shape))
        parts.append(a.reshape(-1))
    out["kinds"], out["shapes"] = kinds, shapes
    out["blob"] = torch.from_numpy(np.concatenate(parts))
    if "cam" in batch[0]:
        out["cam_shapes"] = [tuple(b["cam"].shape) for b in batch]
        out["cam_blob"] = torch.cat([b["cam"].reshape(-1) for b in batch])
        out["cam_keys"] = torch.cat([b["cam_keys"].reshape(-1) for b in batch])
    return out


def split_chunk(chunk):
    """The packs `collate_one` would have produced for the items of a `collate_chunk` message, in order."""
    o = co = ko = 0
    for i, name in enumerate(chunk["names"]):
        shape = chunk["shapes"][i]
        n = int(np.prod(shape))
        pack = {"name": [name], "size": chunk["sizes"][i], "label": chunk["label"][i:i + 1]}
        view = chunk["blob"][o:o + n]
        pack[chunk["kinds"][i]] = view if chunk["kinds"][i] == "jpeg_exact" else view.view((1,) + shape)
        o += n
        if "cam_blob" in chunk:
            cs = chunk["cam_shapes"][i]
            cn = int(np.prod(cs))
            pack["cam"] = chunk["cam_blob"][co:co + cn].view((1,) + cs)
            pack["cam_keys"] = chunk["cam_keys"][ko:ko + cs[0]].view(1, -1)
            co += cn
            ko += cs[0]
        yield pack


def progress(process_id, n_gpus, it, n_items):
    """The reference prints `iter % (len(databin)//20)` which divides by zero for shards < 20 images
    (SURVEY.md D9); same output, guarded."""
    step = max(n_items // 20, 1)
    if process_id == n_gpus - 1 and it % step == 0:
        print("%d " % ((5 * it + 1) // step), end="", flush=True)


def device_pyramid(args):
    """--device_pyramid (default on): loader workers only decode; the per-scale rescale / normalise / flip stack of
    voc12/dataloader.py:191-201 is built on the GPU, bit-identical (irn_b200.preprocess)."""
    return bool(getattr(args, "device_pyramid", True))


def device_jpeg(args):
    """--device_jpeg (True or "exact"; False, the default, has the loader workers decode on the host): JPEG file bytes are decoded
    on the GPU by irn_b200.jpeg.ExactJpegDecoder, bit-identical to the host decoder; the workers ship the bytes of the files it
    supports (jpeg.inspect) and decode the others, so a batch may mix both kinds; the steps that take raw images (cam_to_ir_label)
    ship bytes too.  Needs --device_pyramid."""
    return bool(getattr(args, "device_jpeg", False)) and device_pyramid(args)


def step_batch(args):
    """--step_batch N (default 32): images processed together -- of any sizes in make_sem_seg_labels, make_ins_seg_labels and
    cam_to_ir_label, of equal size in make_cam except when a bucket is topped up with smaller images; 1 = the reference's one-image
    loop."""
    return max(1, int(getattr(args, "step_batch", DEFAULT_STEP_BATCH) or 1))


# a bucketed step holds at most this many times --step_batch images in its pending buckets
PENDING_BOUND = 4


def size_key(pack):
    """Bucket key (H, W): exact-decoder bytes and host-decoded pixels of one size share a bucket (the same pixels either way)."""
    return tuple(pack["size"])


class Batcher:
    """Groups a step's items into batches for `per_batch(ctx, packs)`.

    ragged (make_sem_seg_labels and make_ins_seg_labels, whose network runs every image on the padded crop_size canvas, and
    cam_to_ir_label, whose CRF takes images of any sizes in one call): one pending list, flushed every `bsz` items whatever their sizes.
    Otherwise (make_cam, whose CAM forward runs at each image's own size): one bucket per size, flushed when it holds
    `bsz` items; when more than PENDING_BOUND * bsz items wait in all buckets together, the largest bucket is flushed early, so a
    list with many sizes holds a bounded number of items (each keeps its loader chunk's shared memory alive).  finish() flushes
    what is left.  Every item goes into exactly one batch.

    riders (make_cam, whose CAM forward also takes images of different sizes on one canvas): a bucket flushed before it is full
    (by the bound, or by finish(), largest images first) is topped up to `bsz` items with riders, pending items of other sizes
    that fit inside its H x W and cover at least half its area, the smallest buckets first.  Such a batch runs on the bucket's
    canvas, where a rider costs at most twice its own pixels; a full bucket, and so every batch of a one-size list, is as without
    riders."""

    def __init__(self, ctx, per_batch, bsz, ragged, riders=False):
        self.ctx, self.per_batch, self.bsz, self.ragged, self.riders = ctx, per_batch, bsz, ragged, riders and not ragged
        self.buckets = {}
        self.pending = 0

    def add(self, pack):
        key = None if self.ragged else size_key(pack)
        b = self.buckets.setdefault(key, [])
        b.append(pack)
        self.pending += 1
        if len(b) >= self.bsz:
            self._flush(key)
        elif self.pending > PENDING_BOUND * self.bsz:
            self._flush(max(self.buckets, key=lambda k: len(self.buckets[k])))

    def _flush(self, key):
        packs = self.buckets.pop(key)
        if self.riders and len(packs) < self.bsz:
            packs += self._take_riders(key, self.bsz - len(packs))
        self.pending -= len(packs)
        self.per_batch(self.ctx, packs)

    def _take_riders(self, size, n):
        """Up to n pending items of sizes that fit inside `size` = (H, W) with at least half its area, the smallest buckets first."""
        H, W = size
        fits = [k for k in self.buckets if k[0] <= H and k[1] <= W and 2 * k[0] * k[1] >= H * W]
        out = []
        for k in sorted(fits, key=lambda k: len(self.buckets[k])):
            b = self.buckets[k]
            take = b[:n - len(out)]
            out += take
            del b[:len(take)]
            if not b:
                del self.buckets[k]
            if len(out) == n:
                break
        return out

    def finish(self):
        if self.riders:     # the largest images first: every other bucket may still ride with them
            while self.buckets:
                self._flush(max(self.buckets, key=lambda k: (k[0] * k[1], len(self.buckets[k]))))
            return
        for key in list(self.buckets):
            self._flush(key)


def dataset_name(args):
    """--dataset voc12 (default) or coco."""
    name = str(getattr(args, "dataset", "voc12") or "voc12")
    if name not in ("voc12", "coco"):
        raise ValueError("--dataset must be voc12 or coco, got %r" % name)
    return name


def n_classes(args):
    """The class count of the dataset the step runs on: 20 for PASCAL VOC (and the synthetic images), 80 for MS COCO."""
    if dataset_name(args) == "coco":
        from ..coco.dataloader import N_CAT
        return N_CAT
    return voc_data.N_CAT


def make_dataset(args, list_path, scales, cam_dir=None, cam_field="cam", raw_images=False):
    """VOC images from --voc12_root, MS COCO images from --coco_root with --dataset coco, or seeded synthetic ones with --synthetic N.  `cam_dir`: the label steps let the loader
    workers read the stored CAM dicts (batched mode only; the one-image loop reads them itself, like the reference), and ship
    their `cam_field` map.  `raw_images`: a step without a network takes the decoded uint8 images themselves (host decode, as
    the reference's VOC12ImageDataset with img_normal=None), whatever --device_pyramid / --device_jpeg say."""
    if step_batch(args) == 1 or not (device_pyramid(args) or raw_images):
        cam_dir = None
    decode_only = True if raw_images else device_pyramid(args)
    if getattr(args, "synthetic", 0):
        # one id list for ALL steps (the reference reads --train_list in make_cam but --infer_list in the label steps; with
        # synthetic images the later steps must find the .npy files the first one wrote): --synthetic_list, else 2007_%06d
        names = getattr(args, "synthetic_list", None) or None
        if names is not None and not os.path.exists(names):
            raise FileNotFoundError("--synthetic_list %s" % names)
        return voc_data.SyntheticMSF(int(args.synthetic), scales=scales, name_list=names, decode_only=decode_only, cam_dir=cam_dir,
                                     cam_field=cam_field)
    if dataset_name(args) == "coco":
        from ..coco.dataloader import COCOClassificationDatasetMSF
        return COCOClassificationDatasetMSF(list_path, coco_root=args.coco_root, cls_labels_path=args.coco_cls_labels, scales=scales,
                                            decode_only=decode_only, raw_jpeg=device_jpeg(args), cam_dir=cam_dir, cam_field=cam_field)
    return voc_data.VOC12ClassificationDatasetMSF(list_path, voc12_root=args.voc12_root, scales=scales, decode_only=decode_only,
                                                  raw_jpeg=device_jpeg(args), cam_dir=cam_dir, cam_field=cam_field)


_exact_decoders = {}


def decode_exact(pack):
    """A one-image pack holding exact-decoder bytes -> pack['img_u8'] uint8 [1,H,W,3] on the current device (the one-image loop)."""
    if "jpeg_exact" in pack:
        from ..jpeg import ExactJpegDecoder
        dev = torch.device("cuda", torch.cuda.current_device())
        if dev.index not in _exact_decoders:
            _exact_decoders[dev.index] = ExactJpegDecoder(dev)
        pack["img_u8"] = _exact_decoders[dev.index].decode([pack.pop("jpeg_exact")], names=pack["name"])
    return pack


def attach_pyramid(pack, scales):
    """Turn a decode-only item into what the reference's loader yields: pack['img'] = [1,2,3,h,w] per scale (a single
    tensor when there is one scale, voc12/dataloader.py:200-201), already on the current device."""
    decode_exact(pack)
    if "img_u8" not in pack:
        return pack
    pyr = preprocess.msf_batch(pack["img_u8"].cuda(non_blocking=True), scales)
    pack["img"] = pyr[0][None] if len(scales) == 1 else [p[None] for p in pyr]
    return pack


class Writer:
    """File output off the GPU-issuing thread.  A job is `fn(*args)` run on a pool thread after `event` (recorded on the
    compute stream by the submitter) has completed; jobs do their device->host copies on a side stream of their own, so
    they never queue behind the next batch's kernels, and fan the per-image file writes (np.save pickles, PNG encoding: both
    release the GIL for most of their time) out to a second, wider pool.  At most `max_pending` batch jobs and
    `max_files` file writes are in flight (bounds host and device memory held by finished batches); exceptions surface in
    drain()."""

    def __init__(self, device, threads=2, file_threads=None, max_pending=6, max_files=256):
        self.device = device
        if file_threads is None:
            n_gpus = max(torch.cuda.device_count(), 1)
            file_threads = max(4, min(16, (os.cpu_count() or 8) // n_gpus // 2))
        self.pool = ThreadPoolExecutor(max_workers=threads)
        self.file_pool = ThreadPoolExecutor(max_workers=file_threads)
        self.sem = threading.Semaphore(max_pending)
        self.file_sem = threading.Semaphore(max_files)
        self.futures, self.file_futures = [], []
        self.checks = []        # callables the next batch job runs first, e.g. the status check of the batch's exact JPEG decode
        self._lock = threading.Lock()
        self._tls = threading.local()

    def stream(self):
        s = getattr(self._tls, "stream", None)
        if s is None:
            s = torch.cuda.Stream(device=self.device)
            self._tls.stream = s
        return s

    def to_host(self, tensors):
        """Device tensors -> host tensors through this thread's side stream (call from inside a job, i.e. after the
        producing work has completed).  An entry that is a list of tensors is concatenated along dim 0 first -- on the same
        side stream, so the copy is ordered after the concatenation."""
        s = self.stream()
        with torch.cuda.stream(s):
            out = []
            for t in tensors:
                if isinstance(t, (list, tuple)):
                    t = torch.cat(list(t), 0) if len(t) > 1 else t[0]
                out.append(t.to("cpu", non_blocking=True) if t is not None else None)
        s.synchronize()
        return out

    def submit(self, fn, *args):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        checks, self.checks = self.checks, []
        self.sem.acquire()

        def job():
            try:
                with torch.cuda.device(self.device):
                    ev.synchronize()
                    for c in checks:
                        c()
                    fn(*args)
            finally:
                self.sem.release()
        self.futures.append(self.pool.submit(job))
        if len(self.futures) > 256:
            self.futures = [f for f in self.futures if not (f.done() and f.exception() is None)]

    def submit_file(self, fn, *args):
        """One file write (host only) on the wide pool; callable from the main thread or from inside a batch job."""
        self.file_sem.acquire()

        def job():
            try:
                fn(*args)
            finally:
                self.file_sem.release()
        f = self.file_pool.submit(job)
        with self._lock:
            self.file_futures.append(f)
            if len(self.file_futures) > 1024:
                self.file_futures = [x for x in self.file_futures if not (x.done() and x.exception() is None)]

    submit_host = submit_file

    def map(self, fn, items):
        return list(self.file_pool.map(fn, items))

    def drain(self):
        for f in self.futures:
            f.result()
        self.futures = []
        with self._lock:
            files, self.file_futures = self.file_futures, []
        for f in files:
            f.result()

    def close(self):
        self.drain()
        self.pool.shutdown()
        self.file_pool.shutdown()


class StepContext:
    def __init__(self, model, args, device, scales):
        from ..pipeline import PseudoLabelPipeline
        self.model, self.args, self.device, self.scales = model, args, device, tuple(scales)
        self.pipe = None
        if model is not None:      # cam_to_ir_label has no network
            is_cam = hasattr(model, "classifier")
            self.pipe = PseudoLabelPipeline(model if is_cam else None, None if is_cam else model, device, self.scales,
                                            beta=float(getattr(args, "beta", 10)), exp_times=int(getattr(args, "exp_times", 8)))
        self.writer = Writer(device)
        self._flat = {"bufs": [None, None], "done": [None, None], "i": 0}     # pack_images' staging
        self._exact = None
        self._copy_pool = ThreadPoolExecutor(max_workers=4)
        self.phase_seconds = {} if os.environ.get("IRN_STEP_PROFILE") else None     # host time per phase of the batch bodies

    @contextlib.contextmanager
    def phase(self, name):
        """Host-side stopwatch around a phase of a batch body (IRN_STEP_PROFILE only; GPU work is asynchronous, so this is the
        time the main thread spent issuing it or waiting on something)."""
        if self.phase_seconds is None:
            yield
            return
        t = time.perf_counter()
        try:
            yield
        finally:
            self.phase_seconds[name] = self.phase_seconds.get(name, 0.0) + time.perf_counter() - t

    def pack_images(self, packs):
        """The decoded images of a batch of any sizes as ONE flat device uint8 buffer, image i's [H_i,W_i,3] bytes back to back in
        pack order, and the list of (H_i, W_i); for a batch of one size the buffer is the [N,H,W,3] stack.  Host images are staged
        through two alternating pinned buffers that grow to the largest batch (a buffer is rewritten only after the upload that last
        read it has completed).  With --device_jpeg the exact decoder writes the packs that hold file bytes straight into the buffer,
        in one call whatever their sizes, and the host images are copied in after them; the decode's status words are checked by the
        batch's writer job (Writer.checks)."""
        if any("jpeg_exact" in p for p in packs):
            return self._pack_exact(packs)
        sizes = [(int(p["img_u8"].shape[1]), int(p["img_u8"].shape[2])) for p in packs]
        n = sum(3 * h * w for h, w in sizes)
        slot = self._flat
        k = slot["i"]
        slot["i"] ^= 1
        if slot["done"][k] is not None:
            slot["done"][k].synchronize()
        if slot["bufs"][k] is None or slot["bufs"][k].numel() < n:
            slot["bufs"][k] = torch.empty(n, dtype=torch.uint8).pin_memory()
        buf = slot["bufs"][k][:n]
        offs = np.concatenate([[0], np.cumsum([3 * h * w for h, w in sizes])])

        def put(i):
            buf[int(offs[i]):int(offs[i + 1])].copy_(packs[i]["img_u8"].reshape(-1))
        if len(packs) >= 16:
            list(self._copy_pool.map(put, range(len(packs))))
        else:
            for i in range(len(packs)):
                put(i)
        dev = buf.to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        slot["done"][k] = ev
        return dev, sizes

    def _pack_exact(self, packs):
        from ..jpeg import ExactJpegDecoder
        if self._exact is None:
            self._exact = ExactJpegDecoder(self.device)
        sizes = [tuple(p["size"]) for p in packs]
        offs = np.concatenate([[0], np.cumsum([3 * h * w for h, w in sizes])]).astype(np.int64)
        out = torch.empty(int(offs[-1]), dtype=torch.uint8, device=self.device)
        enc = [i for i, p in enumerate(packs) if "jpeg_exact" in p]
        host = [i for i, p in enumerate(packs) if "jpeg_exact" not in p]
        status = self._exact.decode_into([packs[i]["jpeg_exact"] for i in enc], offs[enc], out, [packs[i]["name"][0] for i in enc])
        self.writer.checks.append(status.check)
        if host:
            flat, _ = self.pack_images([packs[i] for i in host])
            o = 0
            for i in host:
                n = int(offs[i + 1] - offs[i])
                out[int(offs[i]):int(offs[i + 1])].copy_(flat[o:o + n], non_blocking=True)
                o += n
        return out, sizes

    def check_decoded(self):
        """Run the pending exact-decode status checks now (for a batch body that has already waited for its results on the host)."""
        checks, self.writer.checks = self.writer.checks, []
        for c in checks:
            c()


def work_loop(process_id, model, dataset, args, per_image, per_batch=None, ragged=False, riders=False):
    """One GPU's share: the reference's `_work(process_id, model, dataset, args)` signature and loop order
    (step/make_cam.py:16-59), with the per-image / per-batch body supplied by the step.  model None: a step without a network
    (cam_to_ir_label), whose items are the decoded images themselves.  ragged: per_batch takes images of any sizes (the label steps
    and cam_to_ir_label); riders: size buckets topped up with smaller images when flushed early (Batcher, make_cam)."""
    shard = dataset[process_id]
    n_gpus = max(torch.cuda.device_count(), 1)
    scales = getattr(getattr(shard, "dataset", shard), "scales", (1.0,))
    bsz = step_batch(args)
    workers = args.num_workers // n_gpus
    batched = not (per_batch is None or bsz == 1 or not (device_pyramid(args) or model is None))
    if batched:     # items travel in chunks (collate_chunk); the workers keep about two buckets' worth of them in flight
        depth = {"prefetch_factor": max(2, -(-2 * bsz // (workers * LOADER_CHUNK)))} if workers > 0 else {}
        loader = DataLoader(shard, shuffle=False, batch_size=LOADER_CHUNK, num_workers=workers, pin_memory=False, collate_fn=collate_chunk, **depth)
    else:
        loader = DataLoader(shard, shuffle=False, num_workers=workers, pin_memory=False, collate_fn=collate_one)
    with torch.no_grad(), torch.cuda.device(process_id):
        if model is not None:
            model.cuda()
        if not batched:
            for it, pack in enumerate(loader):
                per_image(model, attach_pyramid(pack, scales) if model is not None else decode_exact(pack), args)
                progress(process_id, n_gpus, it, len(shard))
            return
        ctx = StepContext(model, args, torch.device("cuda", process_id), scales)
        batcher = Batcher(ctx, per_batch, bsz, ragged, riders)
        prof = os.environ.get("IRN_STEP_PROFILE")          # host-side time split of the loop (development aid), printed to stderr
        t_load = t_body = 0.0
        t_start = t_prev = time.perf_counter()
        try:
            it = 0
            for msg in loader:
                t_now = time.perf_counter()
                t_load += t_now - t_prev
                for pack in split_chunk(msg):
                    batcher.add(pack)
                    progress(process_id, n_gpus, it, len(shard))
                    it += 1
                t_prev = time.perf_counter()
                t_body += t_prev - t_now
            batcher.finish()
            t_loop = time.perf_counter()
            torch.cuda.synchronize()
            t_sync = time.perf_counter()
        finally:
            ctx.writer.close()
            ctx._copy_pool.shutdown()
        if prof:
            import sys
            t_end = time.perf_counter()
            print("[irn_b200 step profile] rank %d: %d images, %.2f s total = waiting for the loader %.2f + batch bodies (host) %.2f + "
                  "GPU drain %.2f + file writes drain %.2f" % (process_id, len(shard), t_end - t_start, t_load, t_body, t_sync - t_loop,
                                                                t_end - t_sync), file=sys.stderr, flush=True)
            print("[irn_b200 step profile] rank %d: batch-body phases (host seconds): %s" %
                  (process_id, ", ".join("%s %.2f" % kv for kv in sorted(ctx.phase_seconds.items(), key=lambda kv: -kv[1]))), file=sys.stderr, flush=True)


def run_step(args, work, module_name, class_name, weights_path, strict, list_path, scales, opening="[ ", cam_dir=None, cam_field="cam",
             model_kwargs=None):
    """The reference's `run(args)` (e.g. step/make_cam.py:62-77): model class resolved by name (constructed with `model_kwargs`),
    checkpoint loaded, stride partition (misc/torchutils.py:66-68), one process per GPU (a single GPU runs in-process).  module_name
    None: a step without a network (step/cam_to_ir_label.py:44-51); `work` then gets model None and the decoded uint8 images."""
    model = None
    if module_name is not None:
        model = getattr(importlib.import_module(module_name), class_name)(**(model_kwargs or {}))
        model.load_state_dict(torch.load(weights_path), strict=strict)
        model.eval()
    n_gpus = torch.cuda.device_count()
    if n_gpus <= 0:
        raise RuntimeError("irn_b200 steps need at least one CUDA device (there is no CPU fallback)")
    if model is None:
        dataset = make_dataset(args, list_path, scales, cam_dir, cam_field, raw_images=True)
    else:
        dataset = make_dataset(args, list_path, scales, cam_dir)
    shards = torchutils.split_dataset(dataset, n_gpus)
    print(opening, end="")
    if n_gpus == 1:
        work(0, model, shards, args)
    else:
        torch.multiprocessing.spawn(work, nprocs=n_gpus, args=(model, shards, args), join=True)
    print("]")
    torch.cuda.empty_cache()


def load_cam_dicts(ctx, packs, names, cam_out_dir, field="cam"):
    """The stored CAMs of make_cam for a batch (np.load(...).item(), step/make_sem_seg_labels.py:34): what the loader workers
    attached to the items (voc12.dataloader.attach_cam), else read here on the file pool.  Returns (keys list, list of the
    dicts' `field` maps)."""
    if "cam" in packs[0]:
        return [p["cam_keys"][0].numpy() for p in packs], [p["cam"][0] for p in packs]
    stored = ctx.writer.map(lambda n: np.load(os.path.join(cam_out_dir, n + ".npy"), allow_pickle=True).item(), names)
    return [np.asarray(s["keys"]) for s in stored], [s[field] for s in stored]


def to_device_list(ctx, tensors):
    """A list of small host tensors [K_i,h_i,w_i] -> list of device views of ONE uploaded buffer (one H2D copy per batch instead of one
    per image)."""
    tensors = [torch.as_tensor(t) for t in tensors]
    counts = [int(t.numel()) for t in tensors]
    # through PINNED memory (torch's caching host allocator keeps the block alive until the copy has run): a copy from pageable memory
    # is staged in stream order, i.e. the host would sit here until the GPU has finished everything issued before it (the IRNet
    # forward of the same batch)
    staged = torch.empty(sum(counts), dtype=torch.float32, pin_memory=True)
    torch.cat([t.float().reshape(-1) for t in tensors], 0, out=staged)
    dev = staged.to(ctx.device, non_blocking=True)
    out, o = [], 0
    for t, c in zip(tensors, counts):
        out.append(dev[o:o + c].view(t.shape))
        o += c
    return out
