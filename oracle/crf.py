"""Oracle (test infrastructure only): the fully connected CRF of misc/imutils.py:156-170 (crf_inference_label), restated in
numpy float32 from the published algorithm, behind the `pydensecrf` API names the reference calls.

 * mean field  Kraehenbuehl & Koltun, "Efficient Inference in Fully Connected CRFs with Gaussian Edge Potentials", NeurIPS 2011,
               Algorithm 1 and section 4: Q = softmax(-U); each iteration  tmp = -U + sum_m w_m * norm_m (.) L_m(norm_m (.) Q)
               (Potts compatibility: the message of label l only feeds label l, weight = compat), Q = softmax(tmp).
               norm_m = 1/sqrt(L_m(1) + 1e-20): the symmetric normalisation of the filtered kernel (the library default).
 * lattice     Adams, Baek & Davis, "Fast High-Dimensional Filtering Using the Permutohedral Lattice", Eurographics 2010, section 3:
               - 3.1 elevation: feature i scaled by sqrt(2/3)(d+1)/sqrt((i+1)(i+2)) (the per-axis scale that makes the lattice's
                 blur a Gaussian of standard deviation 1 in feature units), mapped onto the hyperplane sum x = 0 of R^{d+1} by
                 E[d] = -d*f[d-1], E[j] = sum_{i>=j} f[i] - j*f[j-1] (evaluated from j = d down to 0 with a running sum);
               - 3.1 enclosing simplex: round every coordinate to the nearest multiple of d+1 (ties to the lower multiple),
                 rank the differences (ties: the earlier coordinate ranks lower), and move the `sum/(d+1)` coordinates of
                 highest (sum > 0) or lowest (sum < 0) rank by -(d+1) / +(d+1) so the point lies on the hyperplane;
               - 3.1 barycentric weights: b[d-rank_i] += (E_i - rem0_i)/(d+1), b[d-rank_i+1] -= the same, b[0] += 1 + b[d+1];
                 vertex r (remainder class r) = rem0 + r - (d+1)*[rank_i > d-r] per coordinate, weight b[r];
               - 3.2 splat: per vertex, the sum of w*value over its pixels in ascending pixel order (sequential float32);
               - 3.2 blur: one pass per lattice direction j = 0..d (in that order), each a Jacobi update
                 v' = v + 0.5*(v[n1] + v[n2]) with n1 = key - 1 + (d+1)e_j, n2 = key + 1 - (d+1)e_j; a neighbour that is not
                 a lattice vertex contributes 0 ([1 2 1]/4 blur, section 3.2, without the 1/4: the constant cancels in the
                 normalisation);
               - 3.2 slice: sum_r ((w_r * v[vertex_r]) * alpha) in r order, alpha = 1/(1 + 2^-d) (the blur's DC gain
                 correction).
               Vertices are stored by their first d coordinates (the last one is minus their sum), packed 64 // d bits each with
               an offset of 2^(bits-1); a coordinate outside that range raises instead of aliasing another vertex.
 * features    Gaussian kernel (x/sxy, y/sxy); bilateral kernel (x/sxy, y/sxy, r/srgb, g/srgb, b/srgb); pixel index y*W + x.
 * step        cam_to_ir_label_one: step/cam_to_ir_label.py:19-41 for one image around crf_inference_q.
 * softmax     subtract the maximum, exp evaluated in float64 and rounded once to float32 (so any correct implementation
               rounds identically), divide by the sequential float32 sum over labels.

Every step is float32 with one rounding per written operation and no fused multiply-add; the CUDA kernels
(irn_b200/csrc/crf.cu) evaluate the same operations in the same order.  Parity with pydensecrf itself is NOT pinned: its sources
are not part of this project and there is no build of it to compare with (DESIGN.md section 2).
"""
import math

import numpy as np

f32 = np.float32


def unary_from_labels(labels, n_labels, gt_prob, zero_unsure=False):
    """pydensecrf.utils.unary_from_labels for zero_unsure=False: U [n_labels, N] float32, -log(gt_prob) for the pixel's label,
    -log((1-gt_prob)/(n_labels-1)) for every other label (computed in float64, rounded once).  n_labels == 1 has no other
    label (the formula's divisor is 0): every entry is -log(gt_prob)."""
    assert not zero_unsure, "only zero_unsure=False is restated"
    labels = np.asarray(labels).reshape(-1)
    if labels.size and (labels.min() < 0 or labels.max() >= n_labels):
        raise ValueError("labels outside [0, %d)" % n_labels)
    p_energy, n_energy = energies(n_labels, gt_prob)
    U = np.full((n_labels, labels.size), n_energy, dtype=np.float32)
    U[labels, np.arange(labels.size)] = p_energy
    return U


def energies(n_labels, gt_prob):
    """(energy of the pixel's own label, energy of every other label) as float32."""
    p = -math.log(gt_prob)
    n = -math.log((1.0 - gt_prob) / (n_labels - 1)) if n_labels > 1 else p
    return f32(p), f32(n)


def scale_factors(d):
    return np.array([(d + 1) * math.sqrt(2.0 / 3.0) / math.sqrt((i + 1) * (i + 2)) for i in range(d)], dtype=np.float32)


def key_bits(d):
    return 64 // d


def pack_keys(k):
    """int64 [M, d] lattice coordinates -> uint64 [M]; raises when a coordinate does not fit."""
    d = k.shape[1]
    bits = key_bits(d)
    off = 1 << (bits - 1)
    b = k + off
    if b.size and (b.min() < 0 or b.max() >= (1 << bits)):
        raise OverflowError("lattice coordinate outside the %d-bit packing range" % bits)
    out = np.zeros(k.shape[0], np.uint64)
    for i in range(d):
        out |= b[:, i].astype(np.uint64) << np.uint64(bits * i)
    return out


def _pack_or_missing(k):
    d = k.shape[1]
    bits = key_bits(d)
    off = 1 << (bits - 1)
    b = k + off
    ok = np.all((b >= 0) & (b < (1 << bits)), axis=1)
    out = np.zeros(k.shape[0], np.uint64)
    bb = np.where(ok[:, None], b, 0)
    for i in range(d):
        out |= bb[:, i].astype(np.uint64) << np.uint64(bits * i)
    return out, ok


def elevate(feat):
    """feat float32 [N, d] -> (elevated float32 [N, d+1], rem0 int64 [N, d+1], rank int64 [N, d+1], bary float32 [N, d+2])."""
    feat = np.asarray(feat, np.float32)
    N, d = feat.shape
    sf = scale_factors(d)
    E = np.zeros((N, d + 1), np.float32)
    sm = np.zeros(N, np.float32)
    for j in range(d, 0, -1):
        cf = feat[:, j - 1] * sf[j - 1]
        E[:, j] = sm - f32(j) * cf
        sm = sm + cf
    E[:, 0] = sm
    down = f32(1.0 / (d + 1))
    dp1 = f32(d + 1)
    v = E * down
    up = np.ceil(v) * dp1
    dn = np.floor(v) * dp1
    rem0f = np.where(up - E < E - dn, up, dn)
    rem0 = rem0f.astype(np.int64)
    s = rem0.sum(1) // (d + 1)
    diff = E - rem0f
    rank = np.zeros((N, d + 1), np.int64)
    for i in range(d + 1):
        for j in range(i + 1, d + 1):
            lt = diff[:, i] < diff[:, j]
            rank[:, i] += lt
            rank[:, j] += ~lt
    sp, sn = s[:, None], s[:, None]
    pos = (s > 0)[:, None]
    neg = (s < 0)[:, None]
    hi = rank >= (d + 1) - sp
    rem0 = np.where(pos & hi, rem0 - (d + 1), rem0)
    rank = np.where(pos, np.where(hi, rank + sp - (d + 1), rank + sp), rank)
    lo = rank < -sn
    rem0 = np.where(neg & lo, rem0 + (d + 1), rem0)
    rank = np.where(neg, np.where(lo, rank + (d + 1) + sn, rank + sn), rank)
    bary = np.zeros((N, d + 2), np.float32)
    rows = np.arange(N)
    for i in range(d + 1):
        val = (E[:, i] - rem0[:, i].astype(np.float32)) * down
        # each slot receives one + and one - term: the sum is the same single rounding in either order
        bary[rows, d - rank[:, i]] += val
        bary[rows, d - rank[:, i] + 1] -= val
    bary[:, 0] = bary[:, 0] + (f32(1) + bary[:, d + 1])
    return E, rem0, rank, bary


def vertex_coords(rem0, rank):
    """Full (d+1)-coordinate keys of the d+1 enclosing vertices: int64 [N, d+1 (vertex r), d+1]."""
    N, dp1 = rem0.shape
    d = dp1 - 1
    r = np.arange(dp1)[None, :, None]
    return rem0[:, None, :] + np.where(rank[:, None, :] <= d - r, r, r - dp1)


class Lattice:
    """A permutohedral lattice over N points with d-dimensional float32 features (Adams et al. 2010, section 3)."""

    def __init__(self, feat):
        feat = np.asarray(feat, np.float32)
        self.N, self.d = feat.shape
        d = self.d
        self.elevated, rem0, rank, bary = elevate(feat)
        self.rem0, self.rank = rem0, rank
        self.weights = bary[:, :d + 1]                                     # [N, d+1]
        self.coords = vertex_coords(rem0, rank)                            # [N, d+1, d+1]
        packed = pack_keys(self.coords[:, :, :d].reshape(-1, d))           # pixel-major: (p, r) pairs in ascending pixel order
        self.keys, inv = np.unique(packed, return_inverse=True)
        self.vertex = inv.reshape(self.N, d + 1).astype(np.int64)          # [N, d+1] vertex id of each (pixel, remainder)
        self.n_vertices = int(self.keys.size)
        # blur neighbours, by binary search among the sorted keys (missing -> index n_vertices, a zero row)
        kc = np.zeros((self.n_vertices, d), np.int64)
        first = np.zeros(self.n_vertices, np.int64)
        first[inv[::-1]] = np.arange(inv.size)[::-1]
        kc[:] = self.coords[:, :, :d].reshape(-1, d)[first]
        self.neighbours = np.zeros((d + 1, 2, self.n_vertices), np.int64)
        for j in range(d + 1):
            for s, sign in enumerate((1, -1)):
                nk = kc - sign
                if j < d:
                    nk[:, j] += sign * (d + 1)
                pk, ok = _pack_or_missing(nk)
                pos = np.minimum(np.searchsorted(self.keys, pk), self.n_vertices - 1)
                hit = ok & (self.keys[pos] == pk)
                self.neighbours[j, s] = np.where(hit, pos, self.n_vertices)
        # splat plan: (pixel, weight) lists per vertex in ascending pixel order, vertices ordered by list length (longest
        # first) so step k of the sequential sum is a contiguous prefix of vertices
        flat = self.vertex.reshape(-1)
        order = np.argsort(flat, kind="stable")                             # stable: ascending pixel within a vertex
        counts = np.bincount(flat, minlength=self.n_vertices)
        starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
        self._by_len = np.argsort(-counts, kind="stable")
        self._len_sorted = counts[self._by_len]
        self._start_sorted = starts[self._by_len]
        self._pair_sorted = order
        self.alpha = f32(1.0 / (1.0 + 2.0 ** (-d)))

    def splat(self, values):
        """values float32 [N, C] -> vertex sums float32 [V, C] (sequential, ascending pixel order)."""
        values = np.asarray(values, np.float32)
        C = values.shape[1]
        d1 = self.d + 1
        pix = self._pair_sorted // d1
        w = self.weights.reshape(-1)[self._pair_sorted]
        acc = np.zeros((self.n_vertices, C), np.float32)
        maxlen = int(self._len_sorted[0]) if self.n_vertices else 0
        # number of vertices whose list is longer than k, for every k
        cnt = np.searchsorted(-self._len_sorted, -(np.arange(maxlen) + 1), side="right")
        for k in range(maxlen):
            m = int(cnt[k])
            idx = self._start_sorted[:m] + k
            acc[self._by_len[:m]] += w[idx, None] * values[pix[idx]]
        return acc

    def blur(self, v):
        v = np.asarray(v, np.float32)
        zero = np.zeros((1, v.shape[1]), np.float32)
        for j in range(self.d + 1):
            vz = np.concatenate([v, zero], 0)
            v = v + f32(0.5) * (vz[self.neighbours[j, 0]] + vz[self.neighbours[j, 1]])
        return v

    def slice(self, v):
        out = np.zeros((self.N, v.shape[1]), np.float32)
        for r in range(self.d + 1):
            out = out + (self.weights[:, r, None] * v[self.vertex[:, r]]) * self.alpha
        return out

    def compute(self, values):
        """L(values): splat, blur, slice.  values float32 [N, C] -> [N, C]."""
        return self.slice(self.blur(self.splat(values)))


def gaussian_features(H, W, sxy):
    y, x = np.mgrid[0:H, 0:W]
    s = f32(sxy)
    return np.stack([x.reshape(-1).astype(np.float32) / s, y.reshape(-1).astype(np.float32) / s], 1)


def bilateral_features(img, sxy, srgb):
    img = np.asarray(img)
    H, W = img.shape[:2]
    g = gaussian_features(H, W, sxy)
    c = img.reshape(-1, 3).astype(np.float32) / f32(srgb)
    return np.concatenate([g, c], 1)


def softmax(x):
    """x float32 [L, N] -> float32 softmax over axis 0: max subtracted, exp in float64 rounded once, sequential sum."""
    x = np.asarray(x, np.float32)
    m = x.max(0)
    e = np.exp((x - m).astype(np.float64)).astype(np.float32)
    s = np.zeros(x.shape[1], np.float32)
    for l in range(x.shape[0]):
        s = s + e[l]
    return e / s


class PairwisePotts:
    def __init__(self, lattice, compat):
        self.lattice = lattice
        self.w = f32(compat)
        one = np.ones((lattice.N, 1), np.float32)
        self.norm = (f32(1) / np.sqrt(lattice.compute(one)[:, 0] + f32(1e-20))).astype(np.float32)

    def message(self, Q):
        """Q float32 [L, N] -> w * norm (.) L(norm (.) Q), float32 [L, N]."""
        f = self.lattice.compute((self.norm[:, None] * Q.T).astype(np.float32))
        return self.w * (self.norm[:, None] * f).T


class DenseCRF2D:
    """pydensecrf.densecrf.DenseCRF2D(W, H, n_labels) with the calls misc/imutils.py:160-168 makes."""

    def __init__(self, W, H, n_labels):
        self.W, self.H, self.n_labels = int(W), int(H), int(n_labels)
        self.U = None
        self.pairwise = []

    def setUnaryEnergy(self, U):
        U = np.asarray(U, np.float32)
        assert U.shape == (self.n_labels, self.W * self.H), U.shape
        self.U = U

    def addPairwiseGaussian(self, sxy=3, compat=3, **kw):
        self.pairwise.append(PairwisePotts(Lattice(gaussian_features(self.H, self.W, sxy)), compat))

    def addPairwiseBilateral(self, sxy=80, srgb=13, rgbim=None, compat=10, **kw):
        rgbim = np.asarray(rgbim)
        assert rgbim.shape == (self.H, self.W, 3) and rgbim.dtype == np.uint8
        self.pairwise.append(PairwisePotts(Lattice(bilateral_features(rgbim, sxy, srgb)), compat))

    def inference(self, t):
        """Q after t mean-field iterations, float32 [n_labels, N]."""
        negU = -self.U
        Q = softmax(negU)
        for _ in range(int(t)):
            tmp = negU
            for p in self.pairwise:
                tmp = tmp + p.message(Q)
            Q = softmax(tmp)
        return Q


def crf_inference_q(img, labels, t=10, n_labels=21, gt_prob=0.7, gauss=(3, 3), bilateral=(50, 5, 10)):
    """Final Q float32 [n_labels, H, W] of crf_inference_label."""
    h, w = img.shape[:2]
    d = DenseCRF2D(w, h, n_labels)
    d.setUnaryEnergy(unary_from_labels(labels, n_labels, gt_prob=gt_prob, zero_unsure=False))
    d.addPairwiseGaussian(sxy=gauss[0], compat=gauss[1])
    d.addPairwiseBilateral(sxy=bilateral[0], srgb=bilateral[1], rgbim=np.ascontiguousarray(np.copy(img)), compat=bilateral[2])
    return d.inference(t).reshape((n_labels, h, w))


def crf_inference_label(img, labels, t=10, n_labels=21, gt_prob=0.7):
    """misc/imutils.py:156-170: argmax over labels of the CRF's Q (first maximum wins)."""
    return np.argmax(crf_inference_q(img, labels, t, n_labels, gt_prob), axis=0)


def cam_to_ir_label_one(img, high_res, keys, fg=0.30, bg=0.05, with_q=False):
    """step/cam_to_ir_label.py:19-41 for one image: img uint8 [H,W,3], high_res fp32 [K,H,W], keys int [K] (make_cam's dict) ->
    dict(conf uint8 [H,W] (the PNG), fg_conf_cam / bg_conf_cam int64 [H,W], pred_fg / pred_bg int64 [H,W], and with `with_q`
    q_fg fp32 [K+1,H,W]).  The CRF is oracle.crf's; n_labels == 1 (no class) gives label 0 everywhere."""
    k = np.pad(np.asarray(keys) + 1, (1, 0), mode="constant")
    cams = np.asarray(high_res, np.float32)
    out = {}
    for tag, thr in (("fg", fg), ("bg", bg)):
        cc = np.argmax(np.pad(cams, ((1, 0), (0, 0), (0, 0)), mode="constant", constant_values=thr), axis=0)
        q = crf_inference_q(img, cc, 10, k.shape[0], 0.7)
        out[tag + "_conf_cam"] = cc
        out["pred_" + tag] = np.argmax(q, axis=0)
        if tag == "fg" and with_q:
            out["q_fg"] = q
    fg_conf, bg_conf = k[out["pred_fg"]], k[out["pred_bg"]]
    conf = fg_conf.copy()
    conf[fg_conf == 0] = 255
    conf[bg_conf + fg_conf == 0] = 0
    out["conf"] = conf.astype(np.uint8)
    return out
