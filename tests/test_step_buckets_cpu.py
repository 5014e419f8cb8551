"""How the batched label steps group their images (irn_b200.step._common.Batcher), without a GPU: the size buckets of make_cam and
cam_to_ir_label stay bounded on a list of many sizes, the size-agnostic steps flush every --step_batch images, and every image is
processed exactly once either way."""
import itertools

import numpy as np
import pytest
import torch

from irn_b200.step import _common


def _packs(sizes):
    return [{"name": ["img%05d" % i], "size": s, "img_u8": torch.empty((1,) + s + (3,), dtype=torch.uint8)} for i, s in enumerate(sizes)]


def _voc_like_sizes(n, seed=0):
    """Mostly 500x375 / 375x500 with a long tail of sizes seen once or twice, in random order."""
    rng = np.random.default_rng(seed)
    common = [(375, 500), (500, 375)]
    tail = [(int(h), int(w)) for h, w in zip(rng.integers(100, 501, n), rng.integers(100, 501, n))]
    return [common[int(rng.integers(2))] if rng.random() < 0.7 else tail[i] for i in range(n)]


class _Recorder:
    def __init__(self, batcher_of):
        self.batches = []
        self.max_pending = 0
        self.batcher = batcher_of(self)

    def __call__(self, ctx, packs):
        self.batches.append([p["name"][0] for p in packs])

    def feed(self, packs):
        for p in packs:
            self.batcher.add(p)
            self.max_pending = max(self.max_pending, self.batcher.pending)
        self.batcher.finish()
        return self


@pytest.mark.parametrize("bsz", [2, 4, 32])
def test_buckets_stay_bounded_and_process_every_image_once(bsz):
    packs = _packs(_voc_like_sizes(1500))
    rec = _Recorder(lambda r: _common.Batcher(None, r, bsz, ragged=False)).feed(packs)
    assert rec.max_pending <= _common.PENDING_BOUND * bsz
    done = list(itertools.chain.from_iterable(rec.batches))
    assert sorted(done) == sorted(p["name"][0] for p in packs) and len(done) == len(set(done))
    size_of = {p["name"][0]: p["size"] for p in packs}
    for b in rec.batches:
        assert 1 <= len(b) <= bsz
        assert len({size_of[n] for n in b}) == 1, "a bucket mixes image sizes"
    assert rec.batcher.pending == 0 and not rec.batcher.buckets


def test_buckets_without_pressure_flush_full_or_at_the_end():
    """Below the bound, a bucket runs when it holds --step_batch images or when the list ends (the behaviour on one-size lists)."""
    sizes = [(64, 96)] * 7 + [(96, 64)] * 3
    rec = _Recorder(lambda r: _common.Batcher(None, r, 4, ragged=False)).feed(_packs(sizes))
    assert [len(b) for b in rec.batches] == [4, 3, 3]


@pytest.mark.parametrize("bsz", [1, 3, 8])
def test_size_agnostic_steps_flush_every_step_batch_images(bsz):
    packs = _packs(_voc_like_sizes(101, seed=1))
    rec = _Recorder(lambda r: _common.Batcher(None, r, bsz, ragged=True)).feed(packs)
    names = [p["name"][0] for p in packs]
    assert rec.batches == [names[i:i + bsz] for i in range(0, len(names), bsz)]
    assert rec.max_pending < bsz
