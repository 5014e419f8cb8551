"""Constructed inputs of the instance-path tests (tests/test_gpu_instance.py), and their premises checked without a GPU: each
case has the property it is built to have, and the oracle's connected components (scipy, standing in for skimage) agree with
an independent breadth-first labeller on every connected-components pattern."""
import collections
import functools

import numpy as np
import pytest

from oracle import steps

# ------------------------------------------------------------------ connected components


def _spiral(h, w):
    """1-pixel-wide square spiral from the top-left corner inwards, arms one pixel apart: one path through half the image,
    so one component whose union-find chains are as long as the image is large."""
    a = np.zeros((h, w), np.int32)
    dirs = ((0, 1), (1, 0), (0, -1), (-1, 0))
    y = x = d = turns = 0
    a[0, 0] = 1

    def free(y1, x1):   # inside, and no foreground 4-neighbour but the pixel it is entered from
        return 0 <= y1 < h and 0 <= x1 < w and not any(
            0 <= y1 + ey < h and 0 <= x1 + ex < w and (y1 + ey, x1 + ex) != (y, x) and a[y1 + ey, x1 + ex] for ey, ex in dirs)

    while turns < 2:
        dy, dx = dirs[d]
        y1, x1 = y + dy, x + dx
        if free(y1, x1) and not a[y1, x1]:
            y, x, turns = y1, x1, 0
            a[y, x] = 1
        else:
            d, turns = (d + 1) % 4, turns + 1
    return a


def _serpentine(h, w):
    """Every even row, joined to the next at alternating ends: one boustrophedon path."""
    a = np.zeros((h, w), np.int32)
    a[0::2] = 1
    a[1::4, w - 1] = 1
    a[3::4, 0] = 1
    return a


def _comb(h, w):
    """Every even column, joined only through the bottom row."""
    a = np.zeros((h, w), np.int32)
    a[:, 0::2] = 1
    a[h - 1] = 1
    return a


def _checker(h, w, v=1):
    yy, xx = np.mgrid[0:h, 0:w]
    return np.where((yy + xx) % 2 == 0, v, 0).astype(np.int32)


def _random(h, w, density, values=(1,), seed=0, block=1):
    rng = np.random.default_rng(seed)
    hb, wb = -(-h // block), -(-w // block)
    on = rng.random((hb, wb)) < density
    v = np.asarray(values, np.int64)[rng.integers(0, len(values), (hb, wb))]
    a = np.where(on, v, 0).astype(np.int32)
    return a.repeat(block, 0).repeat(block, 1)[:h, :w]


EXTREME = (2 ** 31 - 1, 2 ** 31 - 2, -2 ** 31, -2 ** 31 + 1, -1, 1)

CC_PATTERNS = {
    "ones_640": lambda: np.ones((640, 640), np.int32),
    "spiral_640": lambda: _spiral(640, 640),
    "serpentine_640": lambda: _serpentine(640, 640),
    "comb_640": lambda: _comb(640, 640),
    "checker_640": lambda: _checker(640, 640),
    "checker_255x257": lambda: _checker(255, 257, -3),
    "stripes_rows_512x640": lambda: np.where((np.arange(512) // 3) % 2 == 0, 5, 7)[:, None].repeat(640, 1).astype(np.int32),
    "stripes_cols_257x640": lambda: np.where(np.arange(640) % 2 == 0, -9, 4)[None].repeat(257, 0).astype(np.int32),
    "rand055_512": lambda: _random(512, 512, 0.55, seed=1),
    "rand059_512": lambda: _random(512, 512, 0.59, seed=2),
    "rand065_512": lambda: _random(512, 512, 0.65, seed=3),
    "rand055_640": lambda: _random(640, 640, 0.55, seed=4),
    "rand059_640": lambda: _random(640, 640, 0.59, seed=5),
    "rand065_640": lambda: _random(640, 640, 0.65, seed=6),
    "extreme_values": lambda: _random(301, 333, 0.85, EXTREME, seed=7),
    "extreme_values_blocks": lambda: _random(301, 333, 0.9, EXTREME, seed=8, block=3),
    "one_pixel": lambda: np.ones((1, 1), np.int32),
    "one_pixel_background": lambda: np.zeros((1, 1), np.int32),
    "row_1x700": lambda: _random(1, 700, 0.7, (1, 2), seed=9),
    "column_700x1": lambda: _random(700, 1, 0.7, (1, 2), seed=10),
    "width255": lambda: _random(131, 255, 0.59, seed=11),
    "width256": lambda: _random(131, 256, 0.59, seed=12),
    "width257": lambda: _random(131, 257, 0.59, seed=13),
    "width257_three_values": lambda: _random(131, 257, 0.75, (1, 2, 3), seed=14),
}


@functools.lru_cache(maxsize=None)
def cc_pattern(name):
    a = CC_PATTERNS[name]()
    a.flags.writeable = False
    return a


def cc_reference(vals):
    """What irn_connected_components promises, from the oracle's labelling: 0 on background, else 1 + the smallest flat index
    of the pixel's component, a component being a 4-connected set of pixels of one non-zero value."""
    out = np.zeros(vals.size, np.int32)
    for v in np.unique(vals[vals != 0]):
        lab = steps.cc_label(vals == v).reshape(-1)
        ids, first = np.unique(lab, return_index=True)
        table = np.zeros(int(ids.max()) + 1, np.int64)
        table[ids] = first
        m = lab > 0
        out[m] = 1 + table[lab[m]]
    return out.reshape(vals.shape)


def bfs_label(vals):
    """Independent 4-connected labelling of equal non-zero values by breadth-first search from each unlabelled pixel in raster
    order: that pixel is its component's first, so every pixel gets 1 + its flat index."""
    h, w = vals.shape
    v = vals.reshape(-1).tolist()
    lab = [0] * (h * w)
    for s in range(h * w):
        if v[s] == 0 or lab[s]:
            continue
        val, lab[s], q = v[s], s + 1, collections.deque([s])
        while q:
            p = q.popleft()
            y, x = divmod(p, w)
            for n, ok in ((p - w, y > 0), (p + w, y < h - 1), (p - 1, x > 0), (p + 1, x < w - 1)):
                if ok and not lab[n] and v[n] == val:
                    lab[n] = s + 1
                    q.append(n)
    return np.array(lab, np.int32).reshape(h, w)


# ------------------------------------------------------------------ clusters

THRES = np.float32(2.5)
JUST_WEAK_X = np.float32(1.9999)


def thres_field(h=64, w=80):
    """Zero displacement (weak) except three column bands: dp = (1.5, 2.0) and (2.0, 1.5), whose strength is sqrt(6.25) = 2.5 =
    thres exactly and so not weak, each splitting the weak region; and (1.5, 1.9999), just weak (2.0 - 1 ulp would still give
    2.5 in float32), which splits nothing.  With centroids that do not move: the strong bucket plus three weak components, four
    instances."""
    dp = np.zeros((2, h, w), np.float32)
    dp[0, :, 20:23], dp[1, :, 20:23] = 1.5, 2.0
    dp[0, :, 40:42], dp[1, :, 40:42] = 2.0, 1.5
    dp[0, :, 60:63], dp[1, :, 60:63] = 1.5, JUST_WEAK_X
    return dp


def checker_weak_field(h=160, w=160):
    """A strong field (|dp| = 5) with every other pixel weak (dp = 0): with centroids that do not move, ceil(h*w/2) single-pixel
    weak components are present, plus the strong bucket."""
    dp = np.empty((2, h, w), np.float32)
    dp[0], dp[1] = 3.0, -4.0
    on = _checker(h, w) != 0
    dp[:, on] = 0
    return dp


def strong_field(h=125, w=94, seed=0):
    """No weak pixel: every strength is at least 2.6, so every centroid falls in the strong bucket, one instance."""
    rng = np.random.default_rng(seed)
    mag = rng.uniform(2.6, 9.0, (h, w))
    ang = rng.uniform(0, 2 * np.pi, (h, w))
    return np.stack([mag * np.sin(ang), mag * np.cos(ang)]).astype(np.float32)


# ------------------------------------------------------------------ centroids


def clip_field(h, w, seed):
    """Half the pixels displaced by h..2h rows and w..2w columns with random signs, the rest by N(0, 1): steps leave the grid
    on all four sides and are clipped to row 0 / h-1 and column 0 / w-1."""
    rng = np.random.default_rng(seed)
    big = rng.random((h, w)) < 0.5
    dy = np.where(big, rng.choice([-1, 1], (h, w)) * rng.uniform(h, 2 * h, (h, w)), rng.normal(0, 1, (h, w)))
    dx = np.where(big, rng.choice([-1, 1], (h, w)) * rng.uniform(w, 2 * w, (h, w)), rng.normal(0, 1, (h, w)))
    return np.stack([dy, dx]).astype(np.float32)


PITCH = 8


def landing_field(h, w, seed):
    """Zero displacement except at the sources, the pixels whose row and column are multiples of 8.  A source moves by +-1.5
    or +-2.5 in each axis, to an exact .5 position none of whose four bilinear neighbours is a source, so it stays there; or it
    jumps 8 pixels along one axis onto another source (an exact integer position, uy == ly and ux == lx), which moves it on.
    h-1 and w-1 are not multiples of 8, so a position clipped to the far edges is not a source either."""
    assert (h - 1) % PITCH and (w - 1) % PITCH
    rng = np.random.default_rng(seed)
    dp = np.zeros((2, h, w), np.float32)
    for y in range(0, h, PITCH):
        for x in range(0, w, PITCH):
            if rng.random() < 0.35:
                dp[rng.integers(2), y, x] = rng.choice([-PITCH, PITCH])
            else:
                dp[:, y, x] = rng.choice([-2.5, -1.5, 1.5, 2.5], 2)
    return dp


def landing_positions(dp, iterations):
    """Exact positions (float64; every value is a multiple of 0.5) after `iterations` steps on a landing_field: at an integer
    position the step is that pixel's displacement, at a fractional one every pixel of the bilinear footprint is zero."""
    h, w = dp.shape[1:]
    cy, cx = (a.astype(np.float64) for a in np.mgrid[0:h, 0:w])
    for _ in range(iterations):
        ly, lx, uy, ux = (np.floor(cy).astype(int), np.floor(cx).astype(int), np.ceil(cy).astype(int), np.ceil(cx).astype(int))
        whole = (ly == uy) & (lx == ux)
        for c in (0, 1):
            foot = np.abs(dp[c][ly, lx]) + np.abs(dp[c][uy, lx]) + np.abs(dp[c][ly, ux]) + np.abs(dp[c][uy, ux])
            assert not foot[~whole].any(), "a fractional position reads a non-zero displacement"
        cy = np.clip(cy + np.where(whole, dp[0][ly, lx], 0), 0, h - 1)
        cx = np.clip(cx + np.where(whole, dp[1][ly, lx], 0), 0, w - 1)
    return cy, cx


LANDING_CASES = [(61, 83, 1), (61, 83, 2), (61, 83, 5), (61, 83, 300), (160, 107, 300)]

# ------------------------------------------------------------------ detections

MAX_FRAGMENT = 40
DETECT_CLASSES = [14, 2, 2, 7, 19, 7, 0, 11, 14]    # class of each index 1..9, repeated like np.repeat(keys, n_instances)
EMPTY_CHANNEL = 5
NAN_CHANNEL = 8


def detect_case(H, W, seed, nan_plane=None):
    """(scores fp32 [9,H,W], index int32 [H,W]) for detect_instance with max_fragment_size =
    detect_max_fragment(H, W).  On images of at least 140 x 215:
      index 1  a frame two pixels wide round the image: one segment touching every border;
      index 2  a 15 x 20 grid of squares alternately 7 x 7 (area 49) and 6 x 6 (area 36, below 40): 300 segments in one channel;
      index 3  isolated 1-pixel fragments;
      index 4  12 x 12 blocks, plus 1-pixel fragments inside other channels' blocks;
      index 5  no pixel at all;
      index 6  blocks whose scores are multiples of 1/4 (tied maxima) and zero on the left half (all-zero segments);
      index 7  rectangles of area 39, 40 (= max_fragment_size, kept) and 41;
      index 8  blocks scored by `nan_plane` (the all-NaN plane of an all-zero walk), NaN from the host if not given;
      index 9  blocks with random scores.
    Smaller images (below 140 x 215) get runs of 1 to 4 pixels of the same channels in raster order."""
    rng = np.random.default_rng(seed)
    C = len(DETECT_CLASSES)
    scores = rng.random((C, H, W)).astype(np.float32)
    if H < 140 or W < 215:
        runs = [(8, 3), (3, 1), (1, 2), (0, 4), (2, 1), (6, 3), (9, 3)]      # (index, length): 17 pixels a cycle
        index = np.resize(np.concatenate([np.full(n, c, np.int32) for c, n in runs]), H * W).reshape(H, W)
    else:
        index = np.zeros((H, W), np.int32)
        hb, wb = -(-(H - 132) // 12), -(-(W - 4) // 12)
        blocks = rng.choice([0, 4, 6, 8, 9], (hb, wb), p=[0.3, 0.2, 0.2, 0.1, 0.2]).astype(np.int32)
        index[130:H - 2, 2:W - 2] = blocks.repeat(12, 0).repeat(12, 1)[:H - 132, :W - 4]
        yy, xx = np.mgrid[0:H, 0:W]
        frag = (yy % 3 == 0) & (xx % 3 == 0) & (yy > 130) & (yy < H - 3) & (xx > 2) & (xx < W - 3)
        index[frag & (rng.random((H, W)) < 0.01)] = 3
        index[frag & (index != 4) & (index != 3) & (rng.random((H, W)) < 0.004)] = 4
        for i in range(15):
            for j in range(20):
                s = 7 if (i + j) % 2 else 6
                index[4 + 8 * i:4 + 8 * i + s, 4 + 8 * j:4 + 8 * j + s] = 2
        index[4:9, 168:176] = 7        # 40
        index[12:15, 168:181] = 7      # 39
        index[24:25, 168:209] = 7      # 41
        index[:2], index[-2:], index[:, :2], index[:, -2:] = 1, 1, 1, 1
        scores[5] = np.floor(scores[5] * 4) / 4
        scores[5][:, :W // 2] = 0
    scores[NAN_CHANNEL - 1] = np.nan if nan_plane is None else nan_plane
    return scores, index


DETECT_SIZES = [(375, 500), (500, 375), (333, 500), (1, 17), (17, 1), (427, 640)]


def detect_max_fragment(H, W):
    """max_fragment_size for detect_case: 40 on the full layout, 2 on the small random maps (1-pixel fragments score 0,
    the rest keep their maxima)."""
    return MAX_FRAGMENT if H >= 140 and W >= 215 else 2

# ------------------------------------------------------------------ premises


@pytest.mark.parametrize("name", sorted(CC_PATTERNS))
def test_oracle_components_match_breadth_first_search(name):
    vals = cc_pattern(name)
    assert np.array_equal(cc_reference(vals), bfs_label(vals))


def test_component_patterns_are_what_they_claim():
    one = lambda name: steps.cc_label(cc_pattern(name)).max() == 1   # noqa: E731
    for name in ("ones_640", "spiral_640", "serpentine_640", "comb_640"):
        assert one(name), name
    for name in ("spiral_640", "serpentine_640", "comb_640"):        # one pixel wide: no 2 x 2 square of foreground
        a = cc_pattern(name) != 0
        assert not (a[1:, 1:] & a[:-1, 1:] & a[1:, :-1] & a[:-1, :-1]).any(), name
        assert 0.45 < a.mean() < 0.55, name
    # the comb's teeth meet only in the bottom row
    assert steps.cc_label(cc_pattern("comb_640")[:-1]).max() == 320
    for name, (h, w) in (("checker_640", (640, 640)), ("checker_255x257", (255, 257))):
        assert steps.cc_label(cc_pattern(name)).max() == -(-h * w // 2)
    for name, n in (("stripes_rows_512x640", -(-512 // 3)), ("stripes_cols_257x640", 640)):
        assert len(np.unique(cc_reference(cc_pattern(name)))) == n    # neighbouring stripes of different values do not merge
        assert (cc_pattern(name) != 0).all()
    # above the percolation threshold (0.593) the largest cluster spans the image
    for name in ("rand065_512", "rand065_640"):
        lab = steps.cc_label(cc_pattern(name))
        big = np.bincount(lab.ravel())[1:].argmax() + 1
        assert (lab[0] == big).any() and (lab[-1] == big).any() and (lab[:, 0] == big).any() and (lab[:, -1] == big).any(), name
    for name in ("extreme_values", "extreme_values_blocks"):
        assert set(np.unique(cc_pattern(name)).tolist()) == set(EXTREME) | {0}


def test_threshold_is_exact_in_float32():
    assert np.float32(1.5) ** 2 + np.float32(2.0) ** 2 == np.float32(6.25)
    assert np.sqrt(np.float32(6.25)) == THRES and np.sqrt(np.float32(6.25)).dtype == np.float32
    dp = thres_field()
    strength = np.sqrt(dp[1] ** 2 + dp[0] ** 2)
    assert strength.dtype == np.float32
    assert (strength[:, 20:23] == THRES).all() and (strength[:, 40:42] == THRES).all()
    assert (strength[:, 60:63] < THRES).all()
    cen = steps.find_centroids(dp, 0)
    assert np.array_equal(cen, np.stack(np.mgrid[0:64, 0:80]))
    assert steps.cluster_map(cen, dp).max() + 1 == 4
    # were 2.5 weak, everything would be one weak region
    assert steps.cluster_map(cen, dp, np.nextafter(THRES, np.float32(3))).max() + 1 == 1


def test_cluster_cases_have_their_instance_counts():
    dp = checker_weak_field()
    assert steps.cluster_map(steps.find_centroids(dp, 0), dp).max() + 1 == 160 * 160 // 2 + 1
    dp = strong_field()
    assert (np.sqrt(dp[1] ** 2 + dp[0] ** 2) >= 2.6).all()
    assert steps.cluster_map(steps.find_centroids(dp, 0), dp).max() == 0


def test_clip_field_clips_at_both_edges():
    for h, w, seed in ((61, 47, 0), (160, 107, 1)):
        dp = clip_field(h, w, seed)
        assert (dp[0] >= h).any() and (dp[0] <= -h).any() and (dp[1] >= w).any() and (dp[1] <= -w).any()
        for its in (1, 300):
            cen = steps.find_centroids(dp, its)
            assert {0, h - 1} <= set(np.unique(cen[0]).tolist()) and {0, w - 1} <= set(np.unique(cen[1]).tolist())


@pytest.mark.parametrize("h,w,its", LANDING_CASES)
def test_landings_hold_in_the_oracle(h, w, its):
    dp = landing_field(h, w, seed=its)
    cy, cx = landing_positions(dp, its)
    got = steps.find_centroids(dp, its)
    assert np.array_equal(got, np.stack([np.round(cy), np.round(cx)]).astype(np.int32))   # np.round: half to even
    half = (cy % 1 == 0.5) | (cx % 1 == 0.5)
    assert half.sum() >= 20
    # half to even and half away from zero disagree on some of them
    away = np.stack([np.floor(cy + 0.5), np.floor(cx + 0.5)]).astype(np.int32)
    assert (away != got).any(axis=0).sum() >= 10
    # some sources jumped onto another source and moved on from there
    jumped = (np.abs(dp) == PITCH).any(0)
    assert jumped.sum() >= 5


@pytest.mark.parametrize("H,W", DETECT_SIZES)
def test_detect_cases_have_their_features(H, W):
    scores, index = detect_case(H, W, seed=H + W)
    if (H, W) == (427, 640):
        assert H * W % 16 == 0
    else:
        assert H * W % 16 != 0       # the last chunk of 16 pixels is partial: both store paths of segment_masks_kernel run
    assert not (index == EMPTY_CHANNEL).any()
    assert np.isnan(scores[NAN_CHANNEL - 1]).all() and (index == NAN_CHANNEL).any()
    ref = steps.detect_instance(scores, steps.one_hot(index, len(DETECT_CLASSES) + 1)[1:], DETECT_CLASSES,
                                max_fragment_size=detect_max_fragment(H, W))
    assert np.isnan(ref["score"]).any() and (ref["score"] == 0).any() and (ref["score"] > 0).any()
    if H < 140:
        return
    area = {c: np.bincount(steps.cc_label(index == c).ravel())[1:] for c in range(1, len(DETECT_CLASSES) + 1)}
    frame = steps.cc_label(index == 1)
    assert frame.max() == 1 and (frame[0] == 1).all() and (frame[-1] == 1).all() and (frame[:, 0] == 1).all() and (frame[:, -1] == 1).all()
    assert len(area[2]) == 300 and (area[2] < MAX_FRAGMENT).any() and (area[2] > MAX_FRAGMENT).any()
    assert len(area[3]) >= 30 and (area[3] == 1).sum() >= 30
    assert (area[4] == 1).sum() >= 5
    assert sorted(area[7].tolist()) == [MAX_FRAGMENT - 1, MAX_FRAGMENT, MAX_FRAGMENT + 1]
    seg6 = steps.cc_label(index == 6)
    peaks = np.array([scores[5][seg6 == i].max() for i in range(1, seg6.max() + 1)])
    assert (peaks == 0).any() and (peaks > 0).any()
    assert (scores[5] == 1.0 - 0.25).sum() > 1 and (scores[5] == 0).sum() > H * W // 2
