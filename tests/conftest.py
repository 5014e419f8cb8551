import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built_lib():
    """The C-ABI library, built on demand (nvcc cross-compiles on a CPU-only box)."""
    import __graft_entry__ as g
    g.build()
    from irn_b200 import _lib
    return _lib.lib()


@pytest.fixture(scope="session")
def cuda_dev(built_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.fail("a -m gpu test was selected but no CUDA device is visible (there is no CPU fallback)")
    return torch.device("cuda:0")


def record(name, **values):
    """Append a measured parity number to gpurun_out/parity_measured.jsonl (comes back from the GPU box; the asserts
    state the bound, this file states how far inside it the run was)."""
    import json
    try:
        d = os.path.join(ROOT, "gpurun_out")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "parity_measured.jsonl"), "a") as f:
            f.write(json.dumps({"test": name, **{k: (float(v) if hasattr(v, "__float__") else v) for k, v in values.items()}}) + "\n")
    except OSError:
        pass


def golden_path(name):
    return os.path.join(GOLDEN, name)


def unpack_masks(g, suffix=""):
    shape = tuple(g["ins_mask_shape" + suffix])
    return np.unpackbits(g["ins_mask" + suffix], axis=-1, count=shape[-1]).astype(bool).reshape(shape)


def check_detections(got, ref_score, ref_mask, ref_class, score_tol=1e-4, pixel_tol=2e-3):
    """Detections as the reference orders them (channel, then raster order of the segment): same count, same classes in
    the same order, scores within `score_tol`, each mask within `pixel_tol` of the image area (boundary pixels of the
    argmax flip at 1e-5 float noise; a flipped pixel can also split off / merge a 1-pixel fragment, which changes the
    count -- then the comparison falls back to the large segments, which carry every non-zero score)."""
    area = ref_mask.shape[1] * ref_mask.shape[2]
    if len(got["score"]) != len(ref_score):
        big_g = [i for i in range(len(got["score"])) if got["mask"][i].sum() >= 0.01 * area]
        big_r = [i for i in range(len(ref_score)) if ref_mask[i].sum() >= 0.01 * area]
        got = {k: np.asarray(v)[big_g] for k, v in got.items()}
        ref_score, ref_mask, ref_class = ref_score[big_r], ref_mask[big_r], ref_class[big_r]
    assert len(got["score"]) == len(ref_score)
    assert np.asarray(got["class"]).tolist() == np.asarray(ref_class).tolist()
    assert np.abs(np.asarray(got["score"], np.float32) - ref_score).max() < score_tol
    worst = max(float((m != r).mean()) for m, r in zip(got["mask"], ref_mask))
    assert worst < pixel_tol, "mask disagreement %g" % worst
    return worst
