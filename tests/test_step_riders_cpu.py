"""make_cam's grouping (irn_b200.step._common.Batcher with riders), without a GPU: size buckets flushed before they are full are
topped up with smaller images that fit inside the bucket's size and cover at least half its area; every image is processed exactly
once, the pending items stay bounded, and a one-size list gives exactly the batches of plain size buckets."""
import itertools

import numpy as np
import pytest
import torch

from irn_b200.step import _common


def _packs(sizes):
    return [{"name": ["img%05d" % i], "size": s, "img_u8": torch.empty((1,) + s + (3,), dtype=torch.uint8)} for i, s in enumerate(sizes)]


def _voc_like_sizes(n, seed=0):
    """Mostly 500x375 / 375x500, a tail of sizes seen once or twice, and a few near-duplicates of the common sizes (riders)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        r = rng.random()
        if r < 0.6:
            out.append([(375, 500), (500, 375)][int(rng.integers(2))])
        elif r < 0.75:
            out.append((int(rng.integers(300, 376)), int(rng.integers(400, 501))))
        else:
            out.append((int(rng.integers(100, 501)), int(rng.integers(100, 501))))
    return out


def _run(packs, bsz, riders):
    batches, most = [], 0
    b = _common.Batcher(None, lambda ctx, ps: batches.append(list(ps)), bsz, ragged=False, riders=riders)
    for p in packs:
        b.add(p)
        most = max(most, b.pending)
    b.finish()
    assert b.pending == 0 and not b.buckets
    return batches, most


@pytest.mark.parametrize("bsz", [2, 4, 32])
@pytest.mark.parametrize("seed", [0, 1])
def test_riders_fit_their_bucket_and_every_image_runs_once(bsz, seed):
    packs = _packs(_voc_like_sizes(1500, seed))
    batches, most = _run(packs, bsz, riders=True)
    assert most <= _common.PENDING_BOUND * bsz
    done = [p["name"][0] for p in itertools.chain.from_iterable(batches)]
    assert sorted(done) == sorted(p["name"][0] for p in packs) and len(done) == len(set(done))
    mixed = 0
    for batch in batches:
        assert 1 <= len(batch) <= bsz
        H, W = batch[0]["size"]         # the seed bucket comes first
        seed_n = sum(1 for p in batch if p["size"] == (H, W))
        assert all(p["size"] == (H, W) for p in batch[:seed_n]), "the seed bucket's images come first"
        for p in batch[seed_n:]:
            h, w = p["size"]
            assert h <= H and w <= W, ("rider larger than its bucket", (h, w), (H, W))
            assert 2 * h * w >= H * W, ("rider below half its bucket's area", (h, w), (H, W))
        mixed += seed_n < len(batch)
    assert mixed > 0, "the list never produced a rider"


@pytest.mark.parametrize("bsz", [1, 3, 4, 32])
@pytest.mark.parametrize("n", [1, 7, 40, 130])
def test_one_size_list_gives_the_batches_of_plain_buckets(bsz, n):
    packs = _packs([(375, 500)] * n)
    with_riders, _ = _run(packs, bsz, riders=True)
    plain, _ = _run(packs, bsz, riders=False)
    assert [[p["name"][0] for p in b] for b in with_riders] == [[p["name"][0] for p in b] for b in plain]


def test_bucket_full_runs_without_riders_and_leftovers_ride_with_larger_images():
    sizes = [(100, 100)] * 4 + [(90, 80)] * 2 + [(50, 50)] + [(100, 100)] * 2
    batches, _ = _run(_packs(sizes), 4, riders=True)
    got = [[p["size"] for p in b] for b in batches]
    # the first full bucket runs alone; at the end the 100x100 leftovers take the 90x80 riders; 50x50 (a quarter) runs alone
    assert got == [[(100, 100)] * 4, [(100, 100)] * 2 + [(90, 80)] * 2, [(50, 50)]]


def test_riders_ignored_by_size_agnostic_batches():
    packs = _packs(_voc_like_sizes(37, seed=3))
    b = []
    batcher = _common.Batcher(None, lambda ctx, ps: b.append([p["name"][0] for p in ps]), 5, ragged=True, riders=True)
    for p in packs:
        batcher.add(p)
    batcher.finish()
    names = [p["name"][0] for p in packs]
    assert b == [names[i:i + 5] for i in range(0, len(names), 5)]
