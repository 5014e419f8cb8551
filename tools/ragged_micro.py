"""Mixed-size batches against size buckets on one GPU (development aid; bench.py is the contract).

On a synthetic list whose sizes follow a VOC-like mix (most images 500x375 or 375x500, a tail of distinct sizes):
  irn    the IRNet forward of the list as ragged batches (EdgeDisplacement.forward_ragged, --step-batch images each, list order) against
         the per-size forwards (scale-1.0 pyramid + forward_batch on each size bucket, --step-batch images at most per call);
  step   make_sem_seg_labels over the list (CAMs from one make_cam run) with size buckets against ragged batches: the same batch body,
         only the grouping differs (irn_b200.step._common.Batcher);
  cam    make_cam's grouping, size buckets against buckets topped up with riders (Batcher(riders=True)): the CAM stage of the batches
         each policy forms (pyramids + cam_stage per one-size batch, cam_ragged_stage per mixed one; forwards counted, canvas pixels
         over image pixels summed over the scales), then the make_cam step over the list with each policy;
  crf    cam_to_ir_label's grouping on a VOC-like and a COCO-like list (long side 640, short side 360-640, 1-6 of 80 classes): the
         size buckets Batcher(ragged=False) forms against ragged batches of --step-batch images in list order.  CRF device time per
         image (the irn_crf_last_ms events of every CRF call, chunks included, summed; and the span between CUDA events around
         the whole list, host synchronisations included; median of 3, the two policies alternated), CRF calls and host
         synchronisations (two per call: the vertex counts of each lattice), then the cam_to_ir_label step over the list with each
         grouping.
Prints one JSON line with images/s, the card, its power limit and max SM clock."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from irn_b200 import preprocess, synth
from irn_b200.irn import EdgeDisplacement


def voc_like_sizes(n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        r = rng.random()
        if r < 0.45:
            out.append((375, 500))
        elif r < 0.8:
            out.append((500, 375))
        else:
            out.append((int(rng.integers(120, 501)), int(rng.integers(120, 501))))
    return out


def coco_like_sizes(n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        short = int(rng.integers(360, 641))
        out.append((640, short) if rng.random() < 0.3 else (short, 640))
    return out


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def irn_bench(sizes, bsz, reps, dev):
    model = EdgeDisplacement()
    model.load_state_dict(synth.irn_state_dict(), strict=False)
    model.eval()
    pool = {}
    imgs = []
    for i, s in enumerate(sizes):     # a few distinct pixel sets per size: the forward does not depend on the content
        key = (s, i % 4)
        if key not in pool:
            pool[key] = torch.from_numpy(synth.image(i, *s)).to(dev)
        imgs.append(pool[key])

    def ragged():
        for i in range(0, len(imgs), bsz):
            model.forward_ragged(imgs[i:i + bsz])

    buckets = {}
    for i, s in enumerate(sizes):
        buckets.setdefault(s, []).append(i)

    def per_size():
        for s, idx in buckets.items():
            for i in range(0, len(idx), bsz):
                x = torch.stack([imgs[k] for k in idx[i:i + bsz]])
                model.forward_batch(preprocess.msf_batch(x, (1.0,))[0])

    with torch.no_grad():
        ragged(), per_size()       # warm-up: plans, workspaces, resize plans of every size
        t_r, t_b = [], []
        for _ in range(reps):      # alternate the two
            t_r.append(timed(ragged, 1))
            t_b.append(timed(per_size, 1))
    return {"images": len(sizes), "distinct_sizes": len(buckets), "ragged_img_s": len(sizes) / float(np.median(t_r)),
            "per_size_img_s": len(sizes) / float(np.median(t_b)), "ragged_forwards": -(-len(sizes) // bsz),
            "per_size_forwards": sum(-(-len(v) // bsz) for v in buckets.values())}


def step_bench(sizes, bsz, reps, workers):
    from irn_b200.step import _common, make_cam, make_sem_seg_labels
    from irn_b200.voc12 import dataloader
    n = len(sizes)
    tmp = tempfile.mkdtemp(prefix="ragged_micro_")
    torch.save(synth.cam_state_dict(), os.path.join(tmp, "cam.pth.pth"))
    torch.save(synth.irn_state_dict(), os.path.join(tmp, "irn.pth"))

    def mixed(a, list_path, scales, cam_dir=None):
        return dataloader.SyntheticMSF(n, scales=scales, decode_only=True, cam_dir=cam_dir, sizes=sizes)

    a = types.SimpleNamespace(num_workers=workers, voc12_root=tmp, train_list="", infer_list="", cam_network="irn_b200.cam",
                              irn_network="irn_b200.irn", cam_scales=(1.0, 0.5, 1.5, 2.0), cam_weights_name=os.path.join(tmp, "cam.pth"),
                              irn_weights_name=os.path.join(tmp, "irn.pth"), beta=10, exp_times=8, sem_seg_bg_thres=0.25, synthetic=n,
                              step_batch=bsz, cam_out_dir=os.path.join(tmp, "cam"), sem_seg_out_dir=os.path.join(tmp, "sem"))
    os.makedirs(a.cam_out_dir)
    os.makedirs(a.sem_seg_out_dir)
    real_make, real_work = _common.make_dataset, make_sem_seg_labels._work

    def work_with(ragged):
        def work(process_id, model, dataset, args):
            _common.work_loop(process_id, model, dataset, args, make_sem_seg_labels.sem_seg_one_image, make_sem_seg_labels.sem_seg_batch,
                              ragged=ragged)
        return work

    _common.make_dataset = mixed
    try:
        make_cam.run(a)
        res = {}
        for tag, ragged in (("bucketed", False), ("ragged", True), ("bucketed", False), ("ragged", True))[:2 * reps]:
            make_sem_seg_labels._work = work_with(ragged)
            torch.cuda.synchronize()
            t = time.perf_counter()
            make_sem_seg_labels.run(a)
            res.setdefault(tag, []).append(n / (time.perf_counter() - t))
    finally:
        _common.make_dataset, make_sem_seg_labels._work = real_make, real_work
    return {"images": n, "workers": workers, "bucketed_img_s": max(res["bucketed"]), "ragged_img_s": max(res["ragged"]),
            "runs_img_s": res}


def cam_batches(sizes, bsz, riders):
    """The batches (lists of list indices) make_cam's Batcher forms on the list, in order."""
    from irn_b200.step import _common
    out = []
    b = _common.Batcher(None, lambda ctx, packs: out.append([p["name"][0] for p in packs]), bsz, ragged=False, riders=riders)
    for i, s in enumerate(sizes):
        b.add({"name": [i], "size": s, "img_u8": types.SimpleNamespace(shape=(1,) + tuple(s) + (3,))})
    b.finish()
    return out


def cam_bench(sizes, bsz, reps, dev):
    from irn_b200.cam import CAM
    from irn_b200.pipeline import PseudoLabelPipeline
    model = CAM()
    model.load_state_dict(synth.cam_state_dict(), strict=True)
    model.eval()
    pipe = PseudoLabelPipeline(model, None, dev)
    pool, imgs = {}, []
    for i, s in enumerate(sizes):
        key = (s, i % 4)
        if key not in pool:
            pool[key] = torch.from_numpy(synth.image(i, *s)).to(dev)
        imgs.append(pool[key])
    rng = np.random.default_rng(1)
    labels = torch.from_numpy((rng.random((len(sizes), 20)) < 0.1).astype(np.float32))
    labels[np.arange(len(sizes)), rng.integers(0, 20, len(sizes))] = 1

    def run(batches):
        for b in batches:
            if len({sizes[k] for k in b}) == 1:
                xs = pipe.pyramids(torch.stack([imgs[k] for k in b]))
                pipe.cam_stage(xs, labels[b], sizes[b[0]])
            else:
                pipe.cam_ragged_stage(torch.cat([imgs[k].reshape(-1) for k in b]), [sizes[k] for k in b], labels[b])

    def counts(batches):
        fwd, canvas, pixels = 0, 0, 0
        for b in batches:
            for s in pipe.scales:
                sub = max(1, int(pipe.cam_sub * (2.0 / s) ** 2))
                for i in range(0, len(b), sub):
                    hw = [sizes[k] if s == 1 else preprocess.rescaled_size(*sizes[k], s) for k in b[i:i + sub]]
                    fwd += 1
                    canvas += max(h for h, _ in hw) * max(w for _, w in hw) * len(hw)
                    pixels += sum(h * w for h, w in hw)
        return fwd, canvas / pixels

    policies = {"buckets": cam_batches(sizes, bsz, False), "riders": cam_batches(sizes, bsz, True)}
    res = {}
    with torch.no_grad():
        for b in policies.values():     # warm-up: plans, workspaces, resize plans of every size
            run(b)
        t = {k: [] for k in policies}
        for _ in range(reps):           # alternate the two
            for k, b in policies.items():
                t[k].append(timed(lambda: run(b), 1))
    for k, b in policies.items():
        fwd, waste = counts(b)
        res[k] = {"cam_stage_img_s": len(sizes) / float(np.median(t[k])), "runs_s": t[k], "batches": len(b),
                  "mixed_batches": sum(len({sizes[i] for i in x}) > 1 for x in b), "forwards": fwd, "canvas_waste": waste}
    return res


def make_cam_bench(sizes, bsz, reps, workers):
    from irn_b200.step import _common, make_cam
    from irn_b200.voc12 import dataloader
    n = len(sizes)
    tmp = tempfile.mkdtemp(prefix="ragged_micro_cam_")
    torch.save(synth.cam_state_dict(), os.path.join(tmp, "cam.pth.pth"))
    a = types.SimpleNamespace(num_workers=workers, voc12_root=tmp, train_list="", cam_network="irn_b200.cam", cam_scales=(1.0, 0.5, 1.5, 2.0),
                              cam_weights_name=os.path.join(tmp, "cam.pth"), synthetic=n, step_batch=bsz, cam_out_dir=os.path.join(tmp, "cam"))
    os.makedirs(a.cam_out_dir)
    real_make, real_work = _common.make_dataset, make_cam._work

    def work_with(riders):
        def work(process_id, model, dataset, args):
            _common.work_loop(process_id, model, dataset, args, make_cam.cam_one_image, make_cam.cam_batch, riders=riders)
        return work

    _common.make_dataset = lambda a, list_path, scales, cam_dir=None: dataloader.SyntheticMSF(n, scales=scales, decode_only=True, sizes=sizes)
    res = {"buckets": [], "riders": []}
    try:
        make_cam._work = work_with(True)
        make_cam.run(a)                 # warm-up
        for _ in range(reps):
            for tag, riders in (("buckets", False), ("riders", True)):
                make_cam._work = work_with(riders)
                torch.cuda.synchronize()
                t = time.perf_counter()
                make_cam.run(a)
                res[tag].append(n / (time.perf_counter() - t))
    finally:
        _common.make_dataset, make_cam._work = real_make, real_work
    return {"images": n, "workers": workers, "buckets_img_s": float(np.median(res["buckets"])),
            "riders_img_s": float(np.median(res["riders"])), "runs_img_s": res}


def crf_inputs(sizes, n_classes, seed=0):
    """Images (a few pixel sets per size), make_cam-style keys and high_res planes, pooled by (size, class count)."""
    rng = np.random.default_rng(seed + 1)
    lo, hi = (1, 4) if n_classes == 20 else (1, 7)
    imgs, highs, keys, pool = [], [], [], {}
    for i, s in enumerate(sizes):
        k = int(rng.integers(lo, hi))
        key = (s, k, i % 2)
        if key not in pool:
            pool[key] = (synth.image(i, *s), synth.u8_to_cam(synth.cam_planes_u8(k, s[0], s[1], i)))
        imgs.append(pool[key][0])
        highs.append(pool[key][1])
        keys.append(np.sort(rng.choice(n_classes, k, replace=False)))
    return imgs, highs, keys


def crf_bench(sizes, n_classes, bsz, reps, dev):
    from irn_b200 import _lib, crf
    imgs, highs, keys = crf_inputs(sizes, n_classes)
    highs_dev = [torch.from_numpy(h).to(dev) for h in highs]
    policies = {"buckets": cam_batches(sizes, bsz, False), "ragged": [list(range(i, min(i + bsz, len(sizes)))) for i in range(0, len(sizes), bsz)]}
    flats = {k: [torch.from_numpy(np.concatenate([imgs[j].reshape(-1) for j in b])).to(dev) for b in v] for k, v in policies.items()}
    calls, timed = {}, [0.0]
    real_check = _lib.check

    def counting_check(rc, what=""):
        real_check(rc, what)
        if what.startswith("irn_ir_label"):      # one CRF call: a batch over the workspace bound is split into several
            calls[what] = calls.get(what, 0) + 1
            timed[0] += sum(crf.last_ms())        # the events of this call (each call overwrites the last call's)

    def run(k):
        """-> (summed device ms of every CRF call, ms between CUDA events around the whole list, CRF calls)."""
        calls.clear()
        timed[0] = 0.0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for b, flat in zip(policies[k], flats[k]):
            if len({sizes[j] for j in b}) == 1:
                x = flat.view((len(b),) + sizes[b[0]] + (3,))
                crf.ir_labels(x, [highs_dev[j] for j in b], [keys[j] for j in b], 0.30, 0.05, n_classes=n_classes)
            else:
                crf.ir_labels_ragged(flat, [sizes[j] for j in b], [highs_dev[j] for j in b], [keys[j] for j in b], 0.30, 0.05,
                                     n_classes=n_classes)
        e1.record()
        torch.cuda.synchronize()
        return timed[0], e0.elapsed_time(e1), sum(calls.values())

    res = {}
    crf.set_timing(True)
    _lib.check = counting_check
    try:
        for k in policies:              # warm-up
            run(k)
        t = {k: [] for k in policies}
        for _ in range(reps):           # alternate the two
            for k in policies:
                t[k].append(run(k))
        for k in policies:
            n_calls = t[k][-1][2]
            res[k] = {"crf_ms_per_image": float(np.median([r[0] for r in t[k]])) / len(sizes),
                      "span_ms_per_image": float(np.median([r[1] for r in t[k]])) / len(sizes),
                      "runs_ms(calls summed, span)": [r[:2] for r in t[k]], "batches": len(policies[k]),
                      "mixed_batches": sum(len({sizes[j] for j in b}) > 1 for b in policies[k]), "crf_calls": n_calls,
                      "host_syncs": 2 * n_calls}
    finally:
        _lib.check = real_check
        crf.set_timing(False)
    return res


def ir_label_step_bench(sizes, n_classes, bsz, reps, workers):
    """cam_to_ir_label over the list (CAM dicts written first) with size buckets and with ragged batches."""
    from irn_b200.step import _common, cam_to_ir_label
    from irn_b200.voc12 import dataloader
    n = len(sizes)
    tmp = tempfile.mkdtemp(prefix="ragged_micro_crf_")
    a = types.SimpleNamespace(num_workers=workers, voc12_root=tmp, train_list="", synthetic=n, step_batch=bsz, conf_fg_thres=0.30,
                              conf_bg_thres=0.05, cam_out_dir=os.path.join(tmp, "cam"), ir_label_out_dir=os.path.join(tmp, "ir"),
                              dataset="voc12")
    os.makedirs(a.cam_out_dir)
    os.makedirs(a.ir_label_out_dir)
    _, highs, keys = crf_inputs(sizes, n_classes)
    for i in range(n):
        np.save(os.path.join(a.cam_out_dir, "2007_%06d.npy" % i), {"keys": keys[i], "high_res": highs[i]})
    real_make, real_work, real_nc = _common.make_dataset, cam_to_ir_label._work, _common.n_classes

    def work_with(ragged):
        def work(process_id, dataset, args):
            _common.work_loop(process_id, None, dataset, args, cam_to_ir_label.ir_label_one_image, cam_to_ir_label.ir_label_batch,
                              ragged=ragged)
        return work

    _common.make_dataset = lambda a, list_path, scales, cam_dir=None, cam_field="cam", raw_images=False: dataloader.SyntheticMSF(
        n, scales=scales, decode_only=True, cam_dir=cam_dir, cam_field=cam_field, sizes=sizes, n_classes=n_classes)
    _common.n_classes = lambda args: n_classes
    res = {"buckets": [], "ragged": []}
    try:
        cam_to_ir_label._work = work_with(True)
        cam_to_ir_label.run(a)          # warm-up
        for _ in range(reps):
            for tag, ragged in (("buckets", False), ("ragged", True)):
                cam_to_ir_label._work = work_with(ragged)
                torch.cuda.synchronize()
                t = time.perf_counter()
                cam_to_ir_label.run(a)
                res[tag].append(n / (time.perf_counter() - t))
    finally:
        _common.make_dataset, cam_to_ir_label._work, _common.n_classes = real_make, real_work, real_nc
    return {"images": n, "workers": workers, "buckets_img_s": float(np.median(res["buckets"])),
            "ragged_img_s": float(np.median(res["ragged"])), "runs_img_s": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512, help="images in the list")
    ap.add_argument("--step-batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1), help="loader workers of the step runs")
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--legs", default="irn,step,cam", help="comma-separated: irn, step (make_sem_seg_labels), cam (make_cam), "
                    "crf (cam_to_ir_label)")
    ap.add_argument("--out", default="", help="also write the JSON line to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "ragged_micro measures on a CUDA device"
    dev = torch.device("cuda:0")
    sizes = voc_like_sizes(a.n)
    legs = set(a.legs.split(","))
    res = {"card": card(), "step_batch": a.step_batch, "distinct_sizes": len(set(sizes))}
    if "irn" in legs:
        res["irn"] = irn_bench(sizes, a.step_batch, max(3, a.reps), dev)
    if "step" in legs and not a.skip_step:
        res["make_sem_seg_labels"] = step_bench(sizes, a.step_batch, min(a.reps, 2), a.workers)
    if "cam" in legs:
        res["cam_stage"] = cam_bench(sizes, a.step_batch, max(3, a.reps), dev)
        emit(res, a.out)        # the step runs take longest: keep what is measured so far
        if not a.skip_step:
            res["make_cam"] = make_cam_bench(sizes, a.step_batch, max(3, a.reps), a.workers)
    if "crf" in legs:
        for tag, lst, nc in (("voc", sizes, 20), ("coco", coco_like_sizes(a.n), 80)):
            res["crf_" + tag] = {"distinct_sizes": len(set(lst)), **crf_bench(lst, nc, a.step_batch, 3, dev)}
            emit(res, a.out)
            if not a.skip_step:
                res["cam_to_ir_label_" + tag] = ir_label_step_bench(lst, nc, a.step_batch, max(1, a.reps), a.workers)
                emit(res, a.out)
    res["card_after"] = card()
    emit(res, a.out)
    print(json.dumps(res), flush=True)


def emit(res, out):
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
