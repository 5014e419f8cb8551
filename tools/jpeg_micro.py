"""JPEG decode timing on batches of seeded synthetic 375x500 / 500x375 files (4:2:0, quality 90, half of each orientation): the exact
device decoder (irn_b200.jpeg.ExactJpegDecoder) split into its four stages with CUDA events and PIL on a pool of host threads, both
on the same files; then make_cam and make_sem_seg_labels over a mixed-size synthetic JPEG list with the host decoder and with
--device_jpeg True, run alternately.  Medians after warm-up.

    python tools/jpeg_micro.py [--batch 32] [--reps 3] [--step_images 128] [--out results.json]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time
import types
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = "nvidia-smi unavailable"
    return q


def files(n, seed=0, sizes=((375, 500), (500, 375))):
    from PIL import Image
    from irn_b200 import synth
    out = []
    for i in range(n):
        b = io.BytesIO()
        Image.fromarray(synth.image(seed + i, *sizes[i % len(sizes)])).save(b, format="JPEG", quality=90, subsampling=2)
        out.append(b.getvalue())
    return out


def timed(fn, reps):
    """median device ms (CUDA events around fn) and median host ms of fn + synchronize"""
    import torch
    dev, host = [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t = time.perf_counter()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        host.append(1e3 * (time.perf_counter() - t))
        dev.append(a.elapsed_time(b))
    return float(np.median(dev)), float(np.median(host))


def decoders(batch, reps):
    import ctypes
    import torch
    from PIL import Image
    from irn_b200 import _lib
    from irn_b200.jpeg import ExactJpegDecoder
    streams = files(batch)
    dev = torch.device("cuda:0")
    exact = ExactJpegDecoder(dev)
    rows = {"files": "%d x (375x500 | 500x375), 4:2:0, quality 90, %.0f KB per file on average" % (batch, np.mean([len(s) for s in streams]) / 1024)}
    for _ in range(3):
        exact.decode_packed(streams)
    stages = []
    _lib.check(_lib.lib().irn_jpeg_exact_set_timing(1))
    for _ in range(reps):
        exact.decode_packed(streams)
        ms = (ctypes.c_float * 4)()
        _lib.check(_lib.lib().irn_jpeg_exact_last_ms(ms))
        stages.append(list(ms))
    _lib.check(_lib.lib().irn_jpeg_exact_set_timing(0))
    med = np.median(np.array(stages), 0)
    d, h = timed(lambda: exact.decode_packed(streams, check=False), reps)
    rows["exact_ms_per_batch"] = {"device": d, "host_wall": h, "unstuff": float(med[0]), "entropy": float(med[1]), "idct": float(med[2]),
                                  "upsample_colour": float(med[3])}
    with ThreadPoolExecutor(8) as pool:
        def pil():
            list(pool.map(lambda s: np.asarray(Image.open(io.BytesIO(s)).convert("RGB")), streams))
        pil()
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            pil()
            t.append(1e3 * (time.perf_counter() - t0))
    rows["pil_8_threads_ms_per_batch"] = float(np.median(t))
    return rows


def steps(n_images, rounds, workers):
    """make_cam then make_sem_seg_labels over a mixed-size JPEG list, host decode vs --device_jpeg True, alternately."""
    import torch
    from irn_b200 import synth
    from irn_b200.step import make_cam, make_sem_seg_labels
    from irn_b200.voc12 import dataloader
    sizes = [(375, 500), (500, 375), (333, 500), (500, 333), (281, 500)]
    root = tempfile.mkdtemp(prefix="jpeg_micro_")
    os.makedirs(os.path.join(root, "JPEGImages"))
    ids, labels = [], {}
    for i, data in enumerate(files(n_images, seed=100, sizes=sizes)):
        name = "2009_%06d" % i
        with open(os.path.join(root, "JPEGImages", name + ".jpg"), "wb") as f:
            f.write(data)
        ids.append(name)
        labels[int(name.replace("_", ""))] = synth.label(i, 2)
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(ids) + "\n")
    dataloader._cls_labels["voc12/cls_labels.npy"] = labels
    os.makedirs(os.path.join(root, "sess"))
    torch.save(synth.cam_state_dict(), os.path.join(root, "sess", "res50_cam.pth.pth"))
    torch.save(synth.irn_state_dict(), os.path.join(root, "sess", "res50_irn.pth"))
    times = {"host": {"make_cam": [], "make_sem_seg_labels": []}, "exact": {"make_cam": [], "make_sem_seg_labels": []}}
    for r in range(rounds + 1):          # round 0 warms up (module loads, kernel caches)
        for tag, dj in (("host", False), ("exact", "exact")):
            out = {k: os.path.join(root, "%s_%d_%s" % (tag, r, k)) for k in ("cam", "sem")}
            for d in out.values():
                os.makedirs(d)
            a = types.SimpleNamespace(num_workers=workers, voc12_root=root, train_list=os.path.join(root, "list.txt"),
                                      infer_list=os.path.join(root, "list.txt"), cam_network="irn_b200.cam", irn_network="irn_b200.irn",
                                      cam_scales=(1.0, 0.5, 1.5, 2.0), cam_weights_name=os.path.join(root, "sess", "res50_cam.pth"),
                                      irn_weights_name=os.path.join(root, "sess", "res50_irn.pth"), cam_out_dir=out["cam"],
                                      sem_seg_out_dir=out["sem"], beta=10, exp_times=8, sem_seg_bg_thres=0.25, synthetic=0, device_jpeg=dj)
            for name, step in (("make_cam", make_cam), ("make_sem_seg_labels", make_sem_seg_labels)):
                t = time.perf_counter()
                step.run(a)
                if r:
                    times[tag][name].append(time.perf_counter() - t)
    return {tag: {k: {"images_per_s": n_images / float(np.median(v)), "seconds": [round(x, 3) for x in v]} for k, v in d.items()}
            for tag, d in times.items()} | {"list": "%d synthetic JPEG files, sizes %s in turn, %d loader workers" % (n_images, sizes, workers)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--step_images", type=int, default=128)
    ap.add_argument("--step_rounds", type=int, default=2)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_micro needs a CUDA device")
    res = {"card": card(), "decode": decoders(a.batch, a.reps)}
    print(json.dumps(res), flush=True)
    if a.step_images:
        res["steps"] = steps(a.step_images, a.step_rounds, a.workers)
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
