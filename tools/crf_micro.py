"""Device CRF timing (irn_b200.crf.dense_crf with G = 2 CRFs per image, i.e. the cam_to_ir_label workload, through irn_ir_label)
with CUDA events after warm-up, on batches of seeded synthetic images, plus an HBM roofline from algorithmic bytes and the numpy
oracle's CPU time on the same inputs.

    python tools/crf_micro.py [--batch 8] [--reps 5] [--oracle 1] [--out results.json]

Roofline bytes per image (fp32 values, int32 indices), per lattice with V vertices, P = N*(d+1) pairs and C = 2*n_labels channels
padded to blocks of 8, per iteration: splat reads the CSR (pair index, weight) and the pixel's norm and Q block (P*(4+4) + P*(4+32)
per block), writes V*32 per block; blur reads the vertex, its two neighbour indices and two neighbour rows and writes the vertex
((d+1) passes of V*(32*4 + 8) per block); slice reads P*(4+4+32) and reads/writes T (N*32*2 per block); softmax reads T and writes
Q (N*C*4*2).  The neighbour rows are usually L2 hits, so this is an upper bound on HBM traffic.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def algorithmic_bytes(N, n_labels, counts, t=10):
    C = 2 * n_labels
    nb = -(-C // 8)
    total = 0.0
    for d, V in zip((2, 5), counts):
        P = N * (d + 1)
        per_block = P * 8 + P * 36 + V * 32 + (d + 1) * V * (32 * 4 + 8) + P * 40 + N * 64
        total += t * nb * per_block
    total += t * N * C * 8
    return total


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle", type=int, default=1, help="also time the numpy oracle on one image per config")
    ap.add_argument("--out", default="", help="also write all rows as one JSON file")
    a = ap.parse_args()
    import torch
    from irn_b200 import crf, synth
    assert torch.cuda.is_available(), "crf_micro measures the device CRF: no CUDA device visible"
    dev = torch.device("cuda:0")
    rows = []
    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0)}
    print(info, flush=True)
    for (H, W) in ((375, 500), (500, 375), (512, 512)):
        imgs = np.stack([synth.image(100 + i, H, W) for i in range(a.batch)])
        x = torch.from_numpy(imgs).to(dev)
        for n_labels in (2, 4, 21):
            K = n_labels - 1
            highs = [synth.u8_to_cam(synth.cam_planes_u8(K, H, W, i)) for i in range(a.batch)]
            keys = [np.arange(K) for _ in range(a.batch)]
            hd = [torch.from_numpy(h).to(dev) for h in highs]
            crf.ir_labels(x, hd, keys, 0.30, 0.05)           # warm-up (module load, allocator)
            torch.cuda.synchronize()
            crf.set_timing(True)
            times, splits = [], []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _, vc = crf.ir_labels(x, hd, keys, 0.30, 0.05, return_counts=True)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
                splits.append(crf.last_ms())
            crf.set_timing(False)
            ms = float(np.median(times))
            per_img = ms / a.batch
            vmean = vc.mean(0)
            nbytes = algorithmic_bytes(H * W, n_labels, vmean)
            row = {"H": H, "W": W, "n_labels": n_labels, "batch": a.batch, "ms_batch_median": ms, "ms_per_image": per_img,
                   "images_per_s": 1000.0 / per_img, "split_ms_last_chunk(build,iters,tail)": splits[-1],
                   "vertices_mean(gauss,bilateral)": vmean.tolist(), "alg_bytes_per_image": nbytes,
                   "alg_GBps": nbytes / (per_img * 1e-3) / 1e9, "hbm_roofline_fraction": nbytes / HBM_BYTES_PER_S / (per_img * 1e-3)}
            if a.oracle and n_labels <= 4:
                from oracle import crf as ocrf
                t0 = time.time()
                ocrf.cam_to_ir_label_one(imgs[0], highs[0], keys[0])
                row["numpy_oracle_cpu_s_per_image"] = time.time() - t0
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"info": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
