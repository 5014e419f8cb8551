"""Mixed-size batches against size buckets on one GPU (development aid; bench.py is the contract).

On a synthetic list whose sizes follow a VOC-like mix (most images 500x375 or 375x500, a tail of distinct sizes):
  irn    the IRNet forward of the list as ragged batches (EdgeDisplacement.forward_ragged, --step-batch images each, list order) against
         the per-size forwards (scale-1.0 pyramid + forward_batch on each size bucket, --step-batch images at most per call);
  step   make_sem_seg_labels over the list (CAMs from one make_cam run) with size buckets against ragged batches: the same batch body,
         only the grouping differs (irn_b200.step._common.Batcher);
  cam    make_cam's grouping, size buckets against buckets topped up with riders (Batcher(riders=True)): the CAM stage of the batches
         each policy forms (pyramids + cam_stage per one-size batch, cam_ragged_stage per mixed one; forwards counted, canvas pixels
         over image pixels summed over the scales), then the make_cam step over the list with each policy.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512, help="images in the list")
    ap.add_argument("--step-batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1), help="loader workers of the step runs")
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--legs", default="irn,step,cam", help="comma-separated: irn, step (make_sem_seg_labels), cam (make_cam)")
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
