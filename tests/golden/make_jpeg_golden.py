"""Writes tests/golden/jpeg_exact.npz: JPEG files encoded by PIL and the pixels PIL decodes from them
(np.asarray(Image.open(f).convert("RGB"))), the reference for the exact device decoder and its oracle (oracle/jpeg.py).

    python tests/golden/make_jpeg_golden.py

Keys: n, libjpeg_turbo (the version PIL decoded with), and per case i: jpeg<i> (uint8 file bytes), pixels<i> (uint8 [H,W,3]),
name<i> (what the case covers).  `cases()` is also what the CPU test re-encodes live when the installed libjpeg-turbo matches."""
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

SUBSAMPLINGS = {0: "444", 1: "422", 2: "420"}


def pattern(kind, h, w, seed):
    """uint8 [h,w,3] test images: synth (irn_b200.synth, smooth regions + noise), noise (uniform), saturated (black / white and
    pure-colour checkerboards with sharp chroma edges, which push the IDCT into its range-limit clamp)."""
    from irn_b200 import synth
    rng = np.random.RandomState(seed)
    if kind == "synth":
        return synth.image(seed, h, w)
    if kind == "noise":
        return rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    yy, xx = np.mgrid[:h, :w]
    cell = 1 + seed % 5
    chk = ((yy // cell + xx // cell) % 2).astype(bool)
    colours = np.array([[0, 0, 0], [255, 255, 255], [255, 0, 0], [0, 0, 255], [0, 255, 0], [255, 255, 0]], np.uint8)
    a, b = colours[seed % 6], colours[(seed + 1 + seed // 6) % 6]
    return np.where(chk[..., None], a, b).astype(np.uint8)


def encode(img, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img).save(b, format="JPEG", **kw)
    return b.getvalue()


def cases():
    """(name, jpeg bytes) for every case of the fixture."""
    out = []
    seed = 0

    def add(name, img, **kw):
        out.append(("%s %dx%d %s" % (name, img.shape[0], img.shape[1], " ".join("%s=%s" % kv for kv in sorted(kw.items()))), encode(img, **kw)))

    # every residue of H and W mod 16, each sampling
    for r in range(16):
        for ss in SUBSAMPLINGS:
            seed += 1
            add("residue", pattern("noise" if r % 2 else "synth", 17 + r, 32 - r, seed), quality=75, subsampling=ss)
    # 1x1 .. 6x6 (chroma planes 1..3 samples wide: the narrow-plane replication), each sampling
    for h in range(1, 7):
        for w in range(1, 7):
            for ss in SUBSAMPLINGS:
                seed += 1
                add("tiny", pattern("noise", h, w, seed), quality=90, subsampling=ss)
    # qualities x table kinds x restart intervals x samplings, saturated patterns
    for q in (50, 75, 95, 100):
        for ss in SUBSAMPLINGS:
            for kw in ({}, {"optimize": True}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1, "optimize": True}):
                seed += 1
                add("saturated", pattern("saturated", 40, 56, seed), quality=q, subsampling=ss, **kw)
                add("synth", pattern("synth", 24, 40, seed), quality=q, subsampling=ss, **kw)
    # greyscale
    for q, kw in ((75, {}), (95, {"optimize": True}), (100, {"restart_marker_blocks": 2})):
        seed += 1
        add("grey", pattern("synth", 37, 45, seed)[..., 1].copy(), quality=q, **kw)
        add("grey saturated", pattern("saturated", 19, 23, seed)[..., 0].copy(), quality=q, **kw)
    # the sizes the steps see
    add("synth", pattern("synth", 120, 168, 901), quality=90, subsampling=2)
    add("synth", pattern("synth", 120, 168, 902), quality=95, subsampling=0, restart_marker_rows=2)
    add("saturated", pattern("saturated", 375, 500, 903), quality=75, subsampling=2)
    add("saturated", pattern("saturated", 500, 375, 904), quality=90, subsampling=1, optimize=True)
    return out


def main():
    from PIL import Image, features
    arrays = {"libjpeg_turbo": np.array(features.version("libjpeg_turbo") or "")}
    cs = cases()
    for i, (name, data) in enumerate(cs):
        arrays["jpeg%d" % i] = np.frombuffer(data, dtype=np.uint8)
        arrays["pixels%d" % i] = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
        arrays["name%d" % i] = np.array(name)
    arrays["n"] = np.array(len(cs))
    path = os.path.join(HERE, "jpeg_exact.npz")
    np.savez_compressed(path, **arrays)
    print("wrote %s: %d cases, %d bytes" % (path, len(cs), os.path.getsize(path)))


if __name__ == "__main__":
    main()
