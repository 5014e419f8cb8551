"""Every convolution path, held to exact results: the wgmma kernels (3xTF32 and f16x3, every N tile, k-block pairing and ring
depth), the SIMT kernel, the tensor-core stem and the K-concatenated conv3 + projection shortcut.

Exact cases.  The tensor-core kernels evaluate every product as a_hi*w_hi + a_lo*w_hi + a_hi*w_lo.  The data below make that
exact: the input channels form two sets, set A with 12-bit integer activations and weights in {-1, 0, 1}, set B with activations
in {-1, 0, 1} and 12-bit integer weights.  Both splits of every operand then reconstruct it exactly (with the host's
per-output-channel power-of-two prescale of the f16x3 weights), a_lo*w_lo is zero for every product, and every partial sum is
an integer (in units of the prescale) below 2^23.  FixedBatchNorm with gamma = 1, mean = 0, var = float32(1 - 1e-5) folds to the
identity (scale 1 + 6.8e-9, below half an fp32 ulp of any 12-bit integer) and an integer beta is the bias.  So SIMT, 3xTF32 and
f16x3 must return the fp64 result bit for bit whatever order the tensor core adds in: a wrong tap, channel, k-block, swizzle row,
ring stage, tile edge or epilogue operand changes an integer.  The CPU tests (`test_exact_premise`) check all of this for every
case the GPU tests run, by emulating the splits in numpy, so a failure on the GPU is the kernel's.

Measured on an H100 80GB HBM3: wgmma returns these integer sums exactly at the planned bound of 2^23 units.

Real-data cases hold the stem and the fused shortcut to the 1e-5 of max|ref| bar of tests/test_gpu_conv.py against fp64 torch,
check batch invariance and determinism (bitwise), and run f16x3 over the activation range its split documents
(2^-14 <= |a| <= 65504, conv_wgmma.cuh)."""
import os
import re
import zlib
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, record

BOUND = 2 ** 23          # every |partial sum| + |bias| + |residual| stays below this many units
N_SM_STANDIN = 132       # the CPU premise checks of the persistence cases use an H100 SXM's SM count; the data do not depend on it


# ----------------------------------------------------------------------------------------------------------- kernel constants
def wg_stages(f16, bn):
    """WgCfg<F16, BN>::kStages, computed from the constants in conv_wgmma.cuh."""
    src = open(os.path.join(ROOT, "irn_b200", "csrc", "conv_wgmma.cuh")).read()
    a_raw = re.search(r"kARaw = F16 \? (\d+) : (\d+);", src)
    b_bytes = re.search(r"kBBytes = BN \* (\d+);", src)
    max_smem = re.search(r"kMaxSmem = (\d+) \* 1024;", src)
    bar = re.search(r"kBarBytes = (\d+);", src)
    stages = re.search(r"kStages = \(kMaxSmem - 1024 - kBarBytes\) / kStageBytes;", src)
    assert a_raw and b_bytes and max_smem and bar and stages, "WgCfg in conv_wgmma.cuh changed: update wg_stages"
    stage_bytes = int(a_raw.group(1 if f16 else 2)) + 2 * bn * int(b_bytes.group(1))
    return (int(max_smem.group(1)) * 1024 - 1024 - int(bar.group(1))) // stage_bytes


# ------------------------------------------------------------------------------------------------------------------ exact data
def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def channel_sets(rng, cin):
    """True = set A (12-bit activations, ternary weights).  Every group of 8 consecutive channels (one 3xTF32 k-step; an f16x3
    k-step is two) holds both sets."""
    a = np.zeros(cin, bool)
    for c0 in range(0, cin, 8):
        n = min(8, cin - c0)
        a[c0 + rng.permutation(n)[: max(1, n // 2)]] = True
    return a


def int_acts(rng, seta, B, H, W):
    """NCHW float32: set A 12-bit integers, half of them odd and >= 2048 in magnitude (both splits give those a nonzero lo
    part), set B in {-1, 0, 1}."""
    x = rng.integers(-1, 2, (B, len(seta), H, W))
    shape = (B, int(seta.sum()), H, W)
    mag = rng.integers(0, 4096, shape) | np.where(rng.random(shape) < 0.5, 2049, 0)
    x[:, seta] = mag * rng.choice([-1, 1], shape)
    return x.astype(np.float32)


def int_weights(rng, seta, cout, k, density=1.0):
    """OIHW float32: set A input channels in {-1, 0, 1}, set B uniform over [-4095, 4095]; a fraction 1 - density is zero."""
    w = rng.integers(-4095, 4096, (cout, len(seta), k, k))
    w[:, seta] = rng.integers(-1, 2, (cout, int(seta.sum()), k, k))
    w[rng.random(w.shape) >= density] = 0
    return w.astype(np.float32)


def int_bn(rng, cout, shift=0):
    """FixedBatchNorm that folds to the identity with an integer bias.  shift > 0 lifts half the channels by `shift`, so that a
    ReLU after a reduction that cannot stay below 2^23 with the lift does not clamp those outputs."""
    beta = rng.integers(-4096, 4097, cout).astype(np.int64)
    if shift:
        beta[rng.permutation(cout)[: cout // 2]] += shift
    return [np.ones(cout, np.float32), beta.astype(np.float32), np.zeros(cout, np.float32),
            np.full(cout, 1 - 1e-5, np.float32)]


def int_res(rng, shape):
    return rng.integers(-4096, 4097, shape).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------ the cases
Conv = namedtuple("Conv", "id cin cout k stride pad B H W res bn relu density")


def _conv_cases(n_sm):
    cases = [
        Conv("tile_5x11_smaller_than_one_tile", 64, 64, 3, 1, 1, 1, 5, 11, True, True, False, 1.0),
        Conv("image_1x1_only_centre_tap", 128, 128, 3, 1, 1, 2, 1, 1, True, False, False, 1.0),
        Conv("odd_37x51_stride2_3x3_ragged", 64, 128, 3, 2, 1, 2, 37, 51, True, True, False, 1.0),
        Conv("odd_33x47_stride2_1x1_ragged_relu", 256, 256, 1, 2, 0, 2, 33, 47, True, True, True, 1.0),
        Conv("cout192_three_bn64_tiles", 64, 192, 3, 1, 1, 2, 20, 24, False, True, False, 1.0),
        Conv("cout384_three_bn128_tiles_nobias", 128, 384, 1, 1, 0, 2, 24, 40, True, False, False, 1.0),
        Conv("long_k4608_3x3x512", 512, 128, 3, 1, 1, 1, 11, 19, True, True, False, 0.75),
        Conv("long_k4608_3x3x512_bn64_relu", 512, 64, 3, 1, 1, 1, 9, 17, False, True, True, 0.75),
        Conv("cin48_simt_only", 48, 64, 3, 1, 1, 2, 13, 21, True, True, False, 1.0),
    ]
    # k-block pairing: KB = 1 (the unpaired tail alone), 2, 3, S and S + 1 for each of the four kernel instances
    seen = set()
    for f16, bn in ((True, 64), (True, 128), (False, 64), (False, 128)):
        s, bk = wg_stages(f16, bn), 64 if f16 else 32
        for kb in (1, 2, 3, s, s + 1):
            if (kb * bk, bn) in seen:
                continue
            seen.add((kb * bk, bn))
            i = len(seen)
            cases.append(Conv("kb%d_of_%s_bn%d_s%d" % (kb, "f16" if f16 else "tf32", bn, s), kb * bk, bn, 1, 1, 0, 1, 20, 36,
                              i % 2 == 0, i % 3 != 0, i % 4 == 0, 1.0))
    # persistent CTAs: one spatial tile per 16 columns, one N tile; some CTAs take one more work item than others, KB is odd
    for items, name in ((n_sm + 1, "nsm_plus_1"), (2 * n_sm + 3, "2nsm_plus_3")):
        cases.append(Conv("persistent_items_%s" % name, 320, 64, 1, 1, 0, 1, 8, 16 * (items - 1) + 9, True, True, False, 1.0))
    return cases


Stem = namedtuple("Stem", "id B H W Hin Win")
STEM_CASES = [
    Stem("64x64_b2", 2, 64, 64, 64, 64),
    Stem("37x50_wo25_ragged", 1, 37, 50, 37, 50),
    Stem("30x41_padded_to_48x48", 2, 30, 41, 48, 48),
    Stem("32x32_b3", 3, 32, 32, 32, 32),
    Stem("7x9", 1, 7, 9, 7, 9),
]

Shortcut = namedtuple("Shortcut", "id planes cin stride B H W")
SHORTCUT_CASES = [   # the ResNet-50 stage configurations (planes, cin, stride) on small odd grids of several tiles each: the first
    # tile's corner is the same pixel at any stride, so a wrong stride shows only in the tiles after it
    Shortcut("layer1_64_64_s1_3x2_tiles", 64, 64, 1, 2, 11, 37),
    Shortcut("layer2_128_256_s2_2x3_tiles", 128, 256, 2, 2, 37, 41),
    Shortcut("layer3_256_512_s2_2x2_tiles", 256, 512, 2, 2, 19, 35),
    Shortcut("layer4_512_1024_s1_2x2_tiles", 512, 1024, 1, 2, 9, 19),
]


def conv_modes(cin, cout, k):
    return [0] + ([1] if cin % 32 == 0 and cout % 64 == 0 and k in (1, 3) else []) + ([2] if cin % 64 == 0 and cout % 64 == 0 and k in (1, 3) else [])


def conv_data(c):
    rng = _rng(c.id)
    seta = channel_sets(rng, c.cin)
    x = int_acts(rng, seta, c.B, c.H, c.W)
    w = int_weights(rng, seta, c.cout, c.k, c.density)
    bn = int_bn(rng, c.cout) if c.bn else None
    Ho, Wo = (c.H + 2 * c.pad - c.k) // c.stride + 1, (c.W + 2 * c.pad - c.k) // c.stride + 1
    res = int_res(rng, (c.B, c.cout, Ho, Wo)) if c.res else None
    return x, w, bn, res


def stem_data(c):
    rng = _rng("stem_" + c.id)
    seta = channel_sets(rng, 3)
    return int_acts(rng, seta, c.B, c.H, c.W), int_weights(rng, seta, 64, 7), int_bn(rng, 64, shift=2 ** 20)


def shortcut_data(c):
    rng = _rng("shortcut_" + c.id)
    Ho, Wo = (c.H - 1) // c.stride + 1, (c.W - 1) // c.stride + 1
    set_t, set_x = channel_sets(rng, c.planes), channel_sets(rng, c.cin)
    t2, x = int_acts(rng, set_t, c.B, Ho, Wo), int_acts(rng, set_x, c.B, c.H, c.W)
    w3, wds = int_weights(rng, set_t, 4 * c.planes, 1), int_weights(rng, set_x, 4 * c.planes, 1)
    return t2, x, w3, wds, int_bn(rng, 4 * c.planes, shift=2 ** 21), int_bn(rng, 4 * c.planes)


# ------------------------------------------------------------------------------------------------------ numpy split emulation
def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def f16_act_split(a):
    """f16_split2: hi = fp16 round-toward-zero (the fp32 value masked to 11 significant bits), lo = fp16(a - hi) rounded to
    nearest."""
    hi = (_bits(a) & np.uint32(0xFFFFE000)).view(np.float32)
    assert np.array_equal(hi.astype(np.float16).astype(np.float32), hi), "hi is not an fp16 value"
    return hi, (a - hi).astype(np.float16).astype(np.float32)


def tf32_split(a):
    """tf32_hi (and the host's weight split): round to nearest, ties away, on the 13 dropped mantissa bits; lo = a - hi in fp32,
    which the tensor core reads as tf32 (low 13 bits dropped)."""
    hi = ((_bits(a).astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)
    lo = (a - hi).astype(np.float32)
    return hi, (_bits(lo) & np.uint32(0xFFFFE000)).view(np.float32)


def f16_weight_split(w):
    """pack_split (f16x3): per output channel, scale by 2^sh so that max |w| lies in [1, 2), then fp16 hi = rn(v),
    lo = rn(v - hi).  Returns (v, hi, lo) in the scaled units."""
    flat = w.reshape(len(w), -1)
    v = np.empty_like(flat)
    for o in range(len(w)):
        mx = float(np.abs(flat[o]).max())
        e = np.frexp(mx)[1] if mx > 0 else 1
        v[o] = np.ldexp(flat[o], 1 - e).astype(np.float32)
    hi = v.astype(np.float16).astype(np.float32)
    lo = (v - hi).astype(np.float16).astype(np.float32)
    return v.reshape(w.shape), hi.reshape(w.shape), lo.reshape(w.shape)


def bn_fold(w, bn):
    """read_conv's fp64 fold: weight * gamma / sqrt(var + 1e-5), bias = beta - mean * scale, each rounded once to fp32."""
    if bn is None:
        return w, None
    ga, be, mu, va = (np.asarray(t, np.float64) for t in bn)
    scale = ga / np.sqrt(va + 1e-5)
    return (w.astype(np.float64) * scale[:, None, None, None]).astype(np.float32), (be - mu * scale).astype(np.float32)


def check_premise(x, w, bn, stride, pad, extra=0.0, stem=False):
    """x NCHW integers, w OIHW integers: the splits are exact, a_lo * w_lo == 0 for every product, every k-step carries lo
    operands, the BN fold is the identity; returns max over outputs of sum |a||w| + |bias| + extra."""
    wf, bias = bn_fold(w, bn)
    assert np.array_equal(wf, w), "the BN fold changed a weight"
    if bias is not None:
        assert np.array_equal(bias, np.asarray(bn[1], np.float32)), "the BN fold changed the bias"
    a_hi, a_lo = f16_act_split(x)
    t_hi, t_lo = tf32_split(x)
    v, w_hi, w_lo = f16_weight_split(w)
    u_hi, u_lo = tf32_split(w)
    assert np.array_equal(a_hi.astype(np.float64) + a_lo, x) and np.array_equal(t_hi.astype(np.float64) + t_lo, x)
    assert np.array_equal(w_hi.astype(np.float64) + w_lo, v) and np.array_equal(u_hi.astype(np.float64) + u_lo, w)
    for name, alo, wlo in (("f16x3", a_lo, w_lo), ("3xtf32", t_lo, u_lo)):
        a_any = (alo != 0).any(axis=(0, 2, 3))          # per input channel
        w_any = (wlo != 0).any(axis=(0, 2, 3))
        assert not (a_any & w_any).any(), "%s: a_lo * w_lo != 0 in some channel" % name
        for c0 in range(0, len(a_any), 8):               # every k-step holds both kinds of lo operand
            assert a_any[c0:c0 + 8].any() and w_any[c0:c0 + 8].any(), "%s: channels %d.. carry no lo operand" % (name, c0)
        if stem:                                          # the stem's k-blocks are filter rows
            assert all((wlo[:, :, r] != 0).any() for r in range(7)), "%s: a filter row carries no lo weight" % name
    s = F.conv2d(torch.from_numpy(np.abs(x)).double(), torch.from_numpy(np.abs(w)).double(), stride=stride, padding=pad)
    if bias is not None:
        s = s + torch.from_numpy(np.abs(bias)).double()[:, None, None]
    return float((s + torch.as_tensor(extra, dtype=torch.float64)).max())


def _shortcut_reference_inputs(c, t2, x, w3, wds):
    """The fused conv as one 1x1 conv: [t2 ; x sampled at the stride] with [W3 | Wds]."""
    return np.concatenate([t2, x[:, :, ::c.stride, ::c.stride]], axis=1), np.concatenate([w3, wds], axis=1)


@pytest.mark.parametrize("kind,case", [("conv", c) for c in _conv_cases(N_SM_STANDIN)] + [("stem", c) for c in STEM_CASES] +
                         [("shortcut", c) for c in SHORTCUT_CASES], ids=lambda v: v if isinstance(v, str) else v.id)
def test_exact_premise(kind, case):
    """What the GPU exact tests rely on, checked without a GPU for each of their cases."""
    if kind == "conv":
        x, w, bn, res = conv_data(case)
        m = check_premise(x, w, bn, case.stride, case.pad, 0.0 if res is None else np.abs(res))
    elif kind == "stem":
        x, w, bn = stem_data(case)
        xp = np.pad(x, ((0, 0), (0, 0), (0, case.Hin - case.H), (0, case.Win - case.W)))
        m = check_premise(xp, w, bn, 2, 3, stem=True)
    else:
        t2, x, w3, wds, bn3, bnds = shortcut_data(case)
        a, wc = _shortcut_reference_inputs(case, t2, x, w3, wds)
        m = check_premise(a, wc, [bn3[0], bn3[1] + bnds[1], bn3[2], bn3[3]], 1, 0)   # fused: one prescale over [W3 | Wds]
        check_premise(t2, w3, bn3, 1, 0)                                            # the two-conv form: each conv alone
        check_premise(x, wds, bnds, case.stride, 0)
    assert m < BOUND, "partial sums reach %g >= 2^23" % m


def test_stage_counts_follow_wgcfg():
    """The k-block pairing cases are derived from these; the kernel's comment states the same numbers."""
    assert [wg_stages(f, bn) for f, bn in ((True, 128), (True, 64), (False, 128), (False, 64))] == [3, 4, 4, 7]


# ------------------------------------------------------------------------------------------------------------------ GPU: exact
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def assert_exact(y, ref, what):
    if not torch.equal(y, ref):
        d = (y.double() - ref.double()).abs()
        raise AssertionError("%s: %d of %d outputs differ from the exact result, max |diff| %g at %s" %
                             (what, int((d != 0).sum()), d.numel(), d.max().item(), np.unravel_index(int(d.argmax()), d.shape)))


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(_conv_cases(N_SM_STANDIN))), ids=[c.id for c in _conv_cases(N_SM_STANDIN)])
def test_conv_exact(cuda_dev, idx):
    from irn_b200.ops import Conv2d
    c = _conv_cases(_n_sm())[idx]
    x, w, bn, res = conv_data(c)
    ref = F.conv2d(_dev(x).double(), _dev(w).double(), stride=c.stride, padding=c.pad)
    if bn is not None:
        ref = ref + _dev(bn[1]).double()[:, None, None]
    if res is not None:
        ref = ref + _dev(res).double()
    ref = _nhwc(F.relu(ref) if c.relu else ref).float()
    conv = Conv2d(w, bn, c.stride, c.pad)
    xd, rd = _nhwc(_dev(x)), None if res is None else _nhwc(_dev(res))
    for mode in conv_modes(c.cin, c.cout, c.k):
        assert_exact(conv(xd, rd, relu=c.relu, mode=mode), ref, "mode %d" % mode)


@pytest.mark.gpu
@pytest.mark.parametrize("c", STEM_CASES, ids=lambda c: c.id)
def test_stem_exact(cuda_dev, c):
    from irn_b200.ops import Stem
    x, w, bn = stem_data(c)
    xp = F.pad(_dev(x).double(), (0, c.Win - c.W, 0, c.Hin - c.H))
    ref = _nhwc(F.relu(F.conv2d(xp, _dev(w).double(), stride=2, padding=3) + _dev(bn[1]).double()[:, None, None])).float()
    stem = Stem(w, bn)
    for mode in (0, 1, 2):
        assert_exact(stem(_dev(x), c.Hin, c.Win, mode=mode), ref, "stem mode %d" % mode)


@pytest.mark.gpu
@pytest.mark.parametrize("c", SHORTCUT_CASES, ids=lambda c: c.id)
def test_shortcut_exact(cuda_dev, c):
    """The fused conv3 + projection shortcut, and the unfused form the network runs without fusion (ds with relu=False, then c3
    with it as the residual) in every mode."""
    from irn_b200.ops import Conv2d, ShortcutConv
    t2, x, w3, wds, bn3, bnds = shortcut_data(c)
    a, wc = _shortcut_reference_inputs(c, t2, x, w3, wds)
    ref = F.conv2d(_dev(a).double(), _dev(wc).double()) + _dev(bn3[1] + bnds[1]).double()[:, None, None]
    ref = _nhwc(F.relu(ref)).float()
    t2d, xd = _nhwc(_dev(t2)), _nhwc(_dev(x))
    assert_exact(ShortcutConv(w3, bn3, wds, bnds, c.stride)(t2d, xd), ref, "fused")
    ds, c3 = Conv2d(wds, bnds, c.stride, 0), Conv2d(w3, bn3, 1, 0)
    for mode in (0, 1, 2):
        assert_exact(c3(t2d, ds(xd, None, relu=False, mode=mode), relu=True, mode=mode), ref, "two convs, mode %d" % mode)


def test_shortcut_refuses_ineligible_shapes(built_lib):
    from irn_b200 import _lib
    from irn_b200.ops import ShortcutConv
    bn = [np.ones(128, np.float32), np.zeros(128, np.float32), np.zeros(128, np.float32), np.ones(128, np.float32)]
    with pytest.raises(_lib.IrnError, match="planes % 64"):
        ShortcutConv(np.zeros((128, 32), np.float32), bn, np.zeros((128, 64), np.float32), bn, 2)


@pytest.mark.gpu
def test_forward_refuses_another_kind_of_handle(cuda_dev):
    """irn_conv_forward, irn_stem_forward and irn_shortcut_conv_forward each take only handles made by their own create call:
    given one of the other two kinds they return kBadArg (-1) and launch nothing, in the default mode 2."""
    from irn_b200 import _lib
    from irn_b200.ops import Conv2d, ShortcutConv, Stem
    bn = [np.ones(256, np.float32), np.zeros(256, np.float32), np.zeros(256, np.float32), np.ones(256, np.float32)]
    ops = {"conv": Conv2d(np.zeros((64, 64, 1, 1), np.float32)), "stem": Stem(np.zeros((64, 3, 7, 7), np.float32)),
           "shortcut": ShortcutConv(np.zeros((256, 64), np.float32), bn, np.zeros((256, 64), np.float32), bn, 1)}
    L, st = _lib.lib(), _lib.stream_ptr()
    buf = torch.zeros(1 << 20, device="cuda")   # holds every operand of a 1 x 16 x 16 call of any kind
    p, ws = _lib.ptr(buf), L.irn_stem_workspace_bytes(1, 16, 16)
    forward = {
        "conv": lambda h: L.irn_conv_forward(h, p, 1, 16, 16, None, p, 1, 2, st),
        "stem": lambda h: L.irn_stem_forward(h, p, 1, 16, 16, 16, 16, p, 2, p, ws, st),
        "shortcut": lambda h: L.irn_shortcut_conv_forward(h, p, p, 1, 16, 16, p, st),
    }
    for call, run in forward.items():
        for kind, op in ops.items():
            if kind == call:
                continue
            launches = L.irn_total_launch_count()
            rc = run(op._h)
            assert rc == -1, "%s forward on a %s handle returned %d: %s" % (call, kind, rc, L.irn_last_error().decode())
            assert L.irn_total_launch_count() == launches, "%s forward on a %s handle launched a kernel" % (call, kind)


# ------------------------------------------------------------------------------------------------------------- GPU: real data
def _real_bn(g, cout):
    return [1 + 0.1 * torch.randn(cout, generator=g), 0.05 * torch.randn(cout, generator=g), 0.1 * torch.randn(cout, generator=g),
            1 + 0.2 * torch.rand(cout, generator=g)]


def _bn64(y, bn):
    ga, be, mu, va = (t.cuda().double() for t in bn)
    return F.batch_norm(y, mu, va, ga, be, training=False, eps=1e-5)


def _rel_err(y, ref):
    return (y.double() - ref.double()).abs().max().item() / ref.abs().max().item()


def _real_stem(g):
    w = torch.randn((64, 3, 7, 7), generator=g) * (2.0 / 147) ** 0.5
    return w, _real_bn(g, 64)


def _real_shortcut(g, planes, cin):
    w3 = torch.randn((4 * planes, planes, 1, 1), generator=g) * (2.0 / planes) ** 0.5
    wds = torch.randn((4 * planes, cin, 1, 1), generator=g) * (2.0 / cin) ** 0.5
    return w3, _real_bn(g, 4 * planes), wds, _real_bn(g, 4 * planes)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_stem_real_vs_fp64(cuda_dev, mode):
    from irn_b200.ops import Stem
    g = torch.Generator().manual_seed(70 + mode)
    w, bn = _real_stem(g)
    x = torch.randn((2, 3, 45, 61), generator=g).cuda()
    ref = _bn64(F.conv2d(F.pad(x.double(), (0, 3, 0, 3)), w.cuda().double(), stride=2, padding=3), bn)
    ref = _nhwc(F.relu(ref)).float()
    y = Stem(w.numpy(), [t.numpy() for t in bn])(x, 48, 64, mode=mode)
    err = _rel_err(y, ref)
    record("stem_real", mode=mode, rel_err=err)
    assert err < 1e-5, "stem mode %d rel err %g" % (mode, err)


@pytest.mark.gpu
@pytest.mark.parametrize("c", SHORTCUT_CASES, ids=lambda c: c.id)
def test_shortcut_real_vs_fp64(cuda_dev, c):
    from irn_b200.ops import ShortcutConv
    g = torch.Generator().manual_seed(c.planes + c.cin)
    w3, bn3, wds, bnds = _real_shortcut(g, c.planes, c.cin)
    Ho, Wo = (c.H - 1) // c.stride + 1, (c.W - 1) // c.stride + 1
    t2 = torch.relu(torch.randn((c.B, c.planes, Ho, Wo), generator=g)).cuda()
    x = torch.relu(torch.randn((c.B, c.cin, c.H, c.W), generator=g)).cuda()
    ref = _bn64(F.conv2d(t2.double(), w3.cuda().double()), bn3) + _bn64(F.conv2d(x.double(), wds.cuda().double(), stride=c.stride), bnds)
    ref = _nhwc(F.relu(ref)).float()
    y = ShortcutConv(w3.numpy(), [t.numpy() for t in bn3], wds.numpy(), [t.numpy() for t in bnds], c.stride)(_nhwc(t2), _nhwc(x))
    err = _rel_err(y, ref)
    record("shortcut_real", case=c.id, rel_err=err)
    assert err < 1e-5, "fused shortcut rel err %g" % err


def _batch_paths():
    paths = [("conv3x3_ragged", m) for m in (0, 1, 2)] + [("conv1x1_s2_bn64", m) for m in (0, 1, 2)]
    return paths + [("stem", m) for m in (0, 1, 2)] + [("shortcut_s2", 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("path,mode", _batch_paths(), ids=lambda v: str(v))
def test_batch_invariant_and_deterministic(cuda_dev, path, mode):
    """Image b of a batch equals the same image run alone, and two identical calls are equal, bit for bit: the steps' "batched ==
    one-image loop" guarantee rests on this."""
    from irn_b200.ops import Conv2d, ShortcutConv, Stem
    g = torch.Generator().manual_seed(5)
    B = 3
    if path == "stem":
        w, bn = _real_stem(g)
        op = Stem(w.numpy(), [t.numpy() for t in bn])
        xs = (torch.randn((B, 3, 37, 50), generator=g).cuda(),)
        run = lambda x: op(x, 40, 56, mode=mode)
    elif path == "shortcut_s2":
        w3, bn3, wds, bnds = _real_shortcut(g, 128, 256)
        op = ShortcutConv(w3.numpy(), [t.numpy() for t in bn3], wds.numpy(), [t.numpy() for t in bnds], 2)
        xs = (torch.randn((B, 10, 12, 128), generator=g).cuda(), torch.randn((B, 19, 23, 256), generator=g).cuda())
        run = op
    else:
        cin, cout, k, s = (128, 128, 3, 1) if path == "conv3x3_ragged" else (256, 192, 1, 2)
        w = torch.randn((cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5
        op = Conv2d(w.numpy(), [t.numpy() for t in _real_bn(g, cout)], s, k // 2)
        xs = (torch.randn((B, 21, 35, cin), generator=g).cuda(),)
        run = lambda x: op(x, None, relu=False, mode=mode)
    y = run(*xs)
    assert torch.equal(y, run(*xs)), "two identical calls differ"
    for b in range(B):
        assert torch.equal(y[b:b + 1], run(*(t[b:b + 1] for t in xs))), "image %d of the batch differs from the image alone" % b


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
def test_f16x3_dynamic_range(cuda_dev, k):
    """f16x3 across the activation range its split is documented for (2^-14 <= |a| <= 65504): log-uniform magnitudes over
    [2^-14, 3e4], random signs, a tenth exact zeros."""
    from irn_b200.ops import Conv2d
    g = torch.Generator().manual_seed(14 + k)
    cin, cout, B, H, W = 128, 128, 2, 19, 29
    mag = torch.exp2(torch.empty((B, cin, H, W)).uniform_(-14, np.log2(3e4), generator=g))
    x = mag * torch.sign(torch.randn((B, cin, H, W), generator=g)) * (torch.rand((B, cin, H, W), generator=g) >= 0.1)
    w = torch.randn((cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5
    bn = _real_bn(g, cout)
    xd = x.cuda()
    ref = _nhwc(_bn64(F.conv2d(xd.double(), w.cuda().double(), padding=k // 2), bn)).float()
    y = Conv2d(w.numpy(), [t.numpy() for t in bn], 1, k // 2)(_nhwc(xd), None, relu=False, mode=2)
    err = _rel_err(y, ref)
    record("f16x3_dynamic_range", k=k, rel_err=err)
    assert err < 1e-5, "f16x3 rel err %g over the documented range" % err
