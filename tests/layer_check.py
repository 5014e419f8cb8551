"""Per-layer checks of the native CAM / IRNet forwards (tests/test_gpu_layers.py, tests/test_layers_cpu.py).

Each layer is recomputed in float64 from the device's own input (a layer tap, include/irn_b200.h) and the state dict, and
compared with the device's output tap element by element, against a bound that scales with the condition of that
element's sum rather than with the tensor's max.

Convolutions.  y = act(w'.x + b' + r), w' = w gamma/sqrt(var+eps), b' = beta - mean gamma/sqrt(var+eps) folded in fp64:

    |y - y64| <= eps * A + extra,      A = |w'|.|x| + |b'| + |r|      (A by a second, absolute-valued fp64 convolution)

u = 2^-24.  The plan stores w' and b' rounded to fp32 (u |w'|.|x| + u |b'|).
  SIMT (mode 0, and the layers the tensor core does not take): one sequential fp32 FMA chain over K, then + b', + r:
      eps = gamma(K + 3),  gamma(n) = n u / (1 - n u)  (any evaluation order of a K-term dot product obeys it).
  Tensor core (3xTF32 in mode 1, f16x3 in mode 2; conv_wgmma.cuh, DESIGN 4.2): a w ~ a_hi w_hi + a_lo w_hi + a_hi w_lo.
    split, per product, relative to |a||w|:
      f16x3   dropped a_lo w_lo: |a_lo| < 2^-10 |a| (a_hi truncated), |w_lo| <= 2^-11 |w| (w_hi rounded): 2^-21;
              a_lo rounded to fp16: 2^-21; w_lo rounded: 2^-22;  fold: 2^-24                                 -> 21 u
      3xTF32  dropped a_lo w_lo: 2^-11 * 2^-11: 2^-22; a_lo, w_lo read by the tensor core at 11 bits: 2^-21 each;
              fold: 2^-24                                                                                 -> 21 u
    one k-block (64 channels f16x3, 32 channels 3xTF32): 4 k-steps x 3 MMAs = 12 wgmma instructions into a fresh
      accumulator.  Products are exact; each instruction adds its k products and the accumulator aligned to the largest
      with ceil(log2(k+1)) guard bits below fp32's and truncates once: <= 2 * 2^-23 of the sum of the magnitudes it adds,
      which is <= the k-block's share of A                                                                   -> 48 u
    KB partial sums added in IEEE fp32 (KB - 1 roundings), x oscale (a power of two: exact), + b', + r        -> (KB + 1) u
      eps = 21 u + 48 u + (KB + 1) u, to first order (times 1 / (1 - (KB + 70) u)).
    f16x3 only, below fp16's normal range (the `extra` term): an activation |a| < 2^-14 has a_hi on the subnormal grid
      (|a - a_hi - a_lo| <= 2^-24), and for |a| < 2^-4 the residual a - a_hi (< 2^-10 |a| < 2^-14) is itself subnormal, so
      a_lo's rounding is 2^-25 absolute instead of 2^-21 |a|.  Likewise a pre-scaled weight v (max |v| of its channel in
      [1, 2)) below 2^-3 has a subnormal lo: 2^-25 absolute, scaled back by oscale.  Hence
      extra = delta * |w'|.1[|x| < 2^-14] + delta_lo * |w'|.1[|x| < 2^-4] + 2^-24 oscale * sum|x|,  delta = 2^-24, delta_lo = 2^-25.
GroupNorm -> bilinear x up -> crop -> ReLU (gn_up_relu_kernel): mean and rstd from fp64 sums, each rounded to fp32; then
  (x - mean) * rstd * gamma + beta in fp32 (4 roundings + 2 for mean / rstd), the bilinear blend (weights exact for up = 2, 4;
  2 products and 2 sums deep: 4 roundings, relative to the blend of magnitudes):  eps = gamma(10) on
  B = bilinear blend of (|x| + |mean|) rstd |gamma| + |beta|.
edge6 / dp7 (conv1x1_smalln_kernel): 160 / 256 channels over 32 lanes (5 / 8 FMAs), 5 butterfly adds, + bias or - shift:
  eps = gamma(11) / gamma(14) on |w|.|x| + |b|.
CAM flip-add: one fp32 add: bit for bit.  Max pool: bit for bit.  Edge tail: sigmoid(e0/2 + e1/2) with expf (2 ulp),
  1 + E and 1 / (.) rounded: |s - s64| <= s (1 - s) (|a| + 5) u + 2 u s.  dp tail: a copy, bit for bit.
"""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
F16_MAX = 65504.0
BN_EPS = 1e-5
LAYERS = (3, 4, 6, 3)
PLANES = (64, 128, 256, 512)
STRIDES = (1, 2, 2, 1)

# tap ids (include/irn_b200.h)
TAP_STEM, TAP_POOL, TAP_BLOCK0, TAP_CAM_CLS, TAP_HEAD0 = 0, 1, 2, 50, 50
TAP_ECAT, TAP_DCAT3, TAP_DCAT2, TAP_DP7A, TAP_ELOG, TAP_DLOG, TAP_COUNT = 62, 63, 64, 65, 66, 67, 68
HEADS = ["fc_edge%d" % i for i in range(1, 6)] + ["fc_dp%d" % i for i in range(1, 8)]
HEAD_GROUPS = [4] * 5 + [8, 16, 16, 16, 16, 16, 16]
HEAD_UP = [1, 1, 2, 4, 4, 1, 1, 1, 2, 2, 2, 1]
# (concat tap, channel offset) each head's GN output lands in
HEAD_DST = [(TAP_ECAT, 32 * i) for i in range(5)] + [(TAP_DCAT2, 0), (TAP_DCAT2, 64), (TAP_DCAT3, 0), (TAP_DCAT3, 256),
                                                     (TAP_DCAT3, 512), (TAP_DCAT2, 192), (TAP_DP7A, 0)]


def gamma(n):
    return n * U / (1 - n * U)


def blocks():
    """(tap index j, state-dict prefix, planes, stride, first) of the 16 bottlenecks in execution order."""
    out, j = [], 0
    for li, (n, planes, s) in enumerate(zip(LAYERS, PLANES, STRIDES), start=1):
        for b in range(n):
            out.append((j, "resnet50.layer%d.%d" % (li, b), planes, s if b == 0 else 1, b == 0))
            j += 1
    return out


def block_tap(j, which):
    return TAP_BLOCK0 + 3 * j + which


def arith(mode, cin, cout, k):
    """Which arithmetic the plan uses for a conv in `mode` (nets.cu run_conv / split_eligible): 'f16', 'tf32' or 'simt'."""
    tc = cout % 64 == 0 and k in (1, 3)
    if mode == 2 and tc and cin % 64 == 0:
        return "f16"
    if mode >= 1 and tc and cin % 32 == 0:
        return "tf32"
    return "simt"


def eps_for(kind, K, KB):
    if kind == "simt":
        return gamma(K + 3)
    return (21 + 48 + KB + 1) * U / (1 - (KB + 70) * U)


def fold(sd, conv, bn):
    """fp64 folded (w' [cout,cin,k,k], b' [cout]) of conv + FixedBatchNorm; b' None without BN."""
    w = sd[conv].double()
    if bn is None:
        return w, None
    s = sd[bn + ".weight"].double() / torch.sqrt(sd[bn + ".running_var"].double() + BN_EPS)
    return w * s.view(-1, 1, 1, 1), sd[bn + ".bias"].double() - sd[bn + ".running_mean"].double() * s


def oscale(w64):
    """The f16x3 epilogue's per-channel factor (nets.cu pack_split) from the fp32-rounded folded weights."""
    mx = w64.float().abs().flatten(1).amax(1).double()
    e = torch.where(mx > 0, torch.floor(torch.log2(mx)) + 1, torch.ones_like(mx))   # frexp exponent
    return torch.pow(2.0, e - 1)


def nchw(t):
    return t.permute(0, 3, 1, 2)


def _ratio(err, bound):
    """max over elements of err / bound, with err == 0 counting as 0 wherever bound is 0"""
    r = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                    torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.max())


def conv_ratio(x, y, parts, relu, mode, residual=None):
    """Worst |y - y64| / bound of one conv layer.  x: list of fp32 NCHW inputs (one per K segment: conv3 + projection
    shortcut is one K-concatenated reduction), parts: list of (w', b', stride, pad) fp64 folded per segment; residual NCHW
    or None; y the device's NHWC output.  Returns (ratio, arithmetic)."""
    z = 0
    A = 0
    extra = 0
    K = KB = 0
    kinds = set()
    os_all = torch.stack([oscale(w) for w, _, _, _ in parts]).amax(0)   # one pre-scale per channel over [W3 | Wds]
    for xi, (w, b, st, pad) in zip(x, parts):
        cout, cin, k, _ = w.shape
        kind = "f16" if mode == 2 and len(x) == 2 else arith(mode, cin, cout, k)
        if k == 7:   # the stem: tensor-core in modes 1 and 2 over 8 (f16x3) / 7 (3xTF32) filter rows of 32
            kind = "simt" if mode == 0 else ("f16" if mode == 2 else "tf32")
        kinds.add(kind)
        x64 = xi.double()
        z = z + F.conv2d(x64, w, b, stride=st, padding=pad)
        A = A + F.conv2d(x64.abs(), w.abs(), None if b is None else b.abs(), stride=st, padding=pad)
        K += cin * k * k
        KB += (4 if mode == 2 else 7) if k == 7 else cin * k * k // (64 if kind == "f16" else 32)
        if kind == "f16":
            ax = x64.abs()
            wa = w.abs()
            extra = extra + 2.0 ** -24 * F.conv2d((ax < 2.0 ** -14).double(), wa, stride=st, padding=pad) \
                + 2.0 ** -25 * F.conv2d((ax < 2.0 ** -4).double(), wa, stride=st, padding=pad) \
                + 2.0 ** -24 * os_all.view(1, -1, 1, 1) * F.conv2d(ax, torch.ones_like(w[:1]), stride=st, padding=pad)
    if residual is not None:
        z = z + residual.double()
        A = A + residual.double().abs()
    if relu:
        z = F.relu(z)
    kind = "simt" if "simt" in kinds else min(kinds)
    eps = eps_for(kind, K, KB)
    bound = eps * A + extra
    err = (nchw(y).double() - z).abs()
    return _ratio(err, bound), kind


def gn_ref(raw, gamma_, beta, groups, up, hd, wd):
    """fp64 GroupNorm -> bilinear x up -> crop (hd, wd) -> ReLU of raw NHWC, and the bound's B."""
    x = nchw(raw).double()
    Bn, C, H, W = x.shape
    xg = x.reshape(Bn, groups, -1)
    mean = xg.mean(-1, keepdim=True)
    var = ((xg - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    g, b = gamma_.double().view(1, -1, 1, 1), beta.double().view(1, -1, 1, 1)
    y = ((xg - mean) * rstd).reshape(Bn, C, H, W) * g + b
    m = (mean.abs() * rstd).expand(-1, -1, xg.shape[-1]).reshape(Bn, C, H, W)
    mag = (x.abs() * rstd.expand(-1, -1, xg.shape[-1]).reshape(Bn, C, H, W) + m) * g.abs() + b.abs()
    if up > 1:
        y = F.interpolate(y, scale_factor=up, mode="bilinear", align_corners=False)
        mag = F.interpolate(mag, scale_factor=up, mode="bilinear", align_corners=False)
    return F.relu(y[..., :hd, :wd]), mag[..., :hd, :wd]


def gn_ratio(raw, gamma_, beta, groups, up, out_slice):
    hd, wd = out_slice.shape[1], out_slice.shape[2]
    y64, mag = gn_ref(raw, gamma_, beta, groups, up, hd, wd)
    err = (nchw(out_slice).double() - y64).abs()
    return _ratio(err, gamma(10) * mag)


def smalln_ratio(x, w, b, y, n_fma):
    """edge6 / dp7: x NHWC, w [N, Cin] fp64, b [N] fp64 added (bias, or minus the mean shift)"""
    x64 = x.double()
    z = x64 @ w.t() + b
    A = x64.abs() @ w.abs().t() + b.abs()
    return _ratio((y.double() - z).abs(), gamma(n_fma + 5 + 1) * A)


def edge_tail_ratio(elog, edge, P, fh, fw):
    e = elog[..., 0].double()
    a = e[0::2, :fh, :fw] / 2 + e[1::2, :fh, :fw].flip(-1) / 2
    s = torch.sigmoid(a)
    bound = s * (1 - s) * (a.abs() + 5) * U + 2 * U * s
    return _ratio((edge[:, 0].double() - s).abs(), bound)


# ---------------------------------------------------------------------------------------------------------- checkpoints
def _hostile_bn(m, g, gain=1.0):
    c = m.num_features
    mag = torch.pow(2.0, -6 + 8 * torch.rand(c, generator=g)) * gain           # |gamma| log-uniform over 8 binades
    u = torch.rand(c, generator=g)
    sign = torch.where(u < 0.10, -1.0, 1.0)                                     # ~10 % negative
    m.weight.data = torch.where((u >= 0.10) & (u < 0.15), torch.zeros(c), sign * mag)   # ~5 % dead
    var = torch.pow(10.0, -4 + 6 * torch.rand(c, generator=g))                  # running_var log-uniform 1e-4 .. 1e2
    m.running_var.data = var
    m.running_mean.data = 3 * torch.randn(c, generator=g) * torch.sqrt(var)     # a few standard deviations
    m.bias.data = 0.5 * torch.randn(c, generator=g) * mag


def _hostile_trunk(trunk, g, gain):
    """BN statistics as above; each conv's output channel o is scaled by sqrt(running_var[o]), as in a trained network
    whose running variance is the variance its conv produces (otherwise the folded scales, which span more than 20
    binades, would blow the residual stream up): the folded weights then span |gamma|'s 8 binades per channel."""
    mods = dict(trunk.named_modules())
    for name, m in mods.items():
        if isinstance(m, torch.nn.BatchNorm2d):
            last = name.endswith("bn3") or name.endswith("downsample.1")
            _hostile_bn(m, g, gain if last else 1.0)
    for name, m in mods.items():
        if isinstance(m, torch.nn.Conv2d):
            fan_in = m.in_channels * m.kernel_size[0] * m.kernel_size[1]
            bn = mods[name[:-5] + "bn" + name[-1] if name.split(".")[-1].startswith("conv") else name[:-1] + "1"]
            w = torch.randn(m.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5
            m.weight.data = w * torch.sqrt(bn.running_var).view(-1, 1, 1, 1)


def hostile_cam_state_dict(seed=7, gain=0.3):
    """Reference-format CAM state dict with BatchNorm statistics as hostile as a trained network's (module docstring of
    tests/test_gpu_layers.py); `gain` scales |gamma| of bn3 and the projection BN so the residual stream stays bounded."""
    from irn_b200 import _params
    g = torch.Generator().manual_seed(seed)
    m = _params.CamParams()
    _hostile_trunk(m.resnet50, g, gain)
    m.classifier.weight.data = 0.01 * torch.randn(m.classifier.weight.shape, generator=g)
    return {k: v.clone() for k, v in m.state_dict().items()}


def hostile_irn_state_dict(seed=8, gain=0.3):
    """The IRNet counterpart: hostile trunk BN, GroupNorm heads with zero and negative gamma and a first group per head
    whose conv weights share an offset, so its mean over the (non-negative) features is much larger than its std."""
    from irn_b200 import _params, synth
    g = torch.Generator().manual_seed(seed)
    m = _params.IrnParams()
    base = synth.irn_state_dict()
    m.load_state_dict(base, strict=False)
    _hostile_trunk(m.resnet50, g, gain)
    for name, mod in m.named_modules():
        if name.startswith("fc_") and isinstance(mod, torch.nn.Conv2d) and name not in ("fc_edge6", "fc_dp7.3"):
            fan_in = mod.in_channels
            w = torch.randn(mod.weight.shape, generator=g) * (1.0 / fan_in) ** 0.5
            gsz = mod.out_channels // (4 if name.startswith("fc_edge") else (8 if name.startswith("fc_dp1") else 16))
            w[:gsz] += 1.0 / fan_in ** 0.5
            mod.weight.data = w
        elif name.startswith("fc_") and isinstance(mod, torch.nn.GroupNorm):
            c = mod.num_channels
            mag = torch.pow(2.0, -3 + 4 * torch.rand(c, generator=g))
            u = torch.rand(c, generator=g)
            mod.weight.data = torch.where(u < 0.05, torch.zeros(c), torch.where(u < 0.15, -mag, mag))
            mod.bias.data = 0.5 * torch.randn(c, generator=g)
    return {k: v.clone() for k, v in m.state_dict().items()}


# ------------------------------------------------------------------------------------------------------------ layer walk
def trunk_layers(sd, taps, x_in, mode):
    """Yields (name, ratio, arithmetic, max |input|) for the stem and the 48 bottleneck convolutions, each recomputed from
    its device input tap.  x_in: the network input NCHW fp32 (on the taps' device), already zero-padded to the canvas."""
    dev = x_in.device
    sdd = {k: v.to(dev) for k, v in sd.items()}
    P = "resnet50."
    w, b = fold(sdd, P + "conv1.weight", P + "bn1")
    r, kind = conv_ratio([x_in], taps[TAP_STEM], [(w, b, 2, 3)], True, mode)
    yield "stem", r, kind, float(x_in.abs().max())
    x = taps[TAP_POOL]
    for j, p, planes, st, first in blocks():
        t1, t2, out = taps[block_tap(j, 0)], taps[block_tap(j, 1)], taps[block_tap(j, 2)]
        w, b = fold(sdd, p + ".conv1.weight", p + ".bn1")
        r, kind = conv_ratio([nchw(x)], t1, [(w, b, 1, 0)], True, mode)
        yield p + ".conv1", r, kind, float(x.abs().max())
        w, b = fold(sdd, p + ".conv2.weight", p + ".bn2")
        r, kind = conv_ratio([nchw(t1)], t2, [(w, b, st, 1)], True, mode)
        yield p + ".conv2", r, kind, float(t1.abs().max())
        w3, b3 = fold(sdd, p + ".conv3.weight", p + ".bn3")
        if first:
            wd, bd = fold(sdd, p + ".downsample.0.weight", p + ".downsample.1")
            r, kind = conv_ratio([nchw(t2), nchw(x)], out, [(w3, b3, 1, 0), (wd, bd, st, 0)], True, mode)
        else:
            r, kind = conv_ratio([nchw(t2)], out, [(w3, b3, 1, 0)], True, mode, residual=nchw(x))
        yield p + ".conv3", r, kind, max(float(t2.abs().max()), float(x.abs().max()))
        x = out


def maxpool_exact(taps):
    ref = F.max_pool2d(nchw(taps[TAP_STEM]), 3, 2, 1).permute(0, 2, 3, 1)
    return bool(torch.equal(ref, taps[TAP_POOL]))


def irn_head_layers(sd, taps, mode):
    """Yields (name, ratio, arithmetic, max |input|) of the 12 head convs, their GroupNorm stages, edge6 and dp7."""
    dev = taps[TAP_POOL].device
    xs = [taps[TAP_POOL]] + [taps[block_tap(j, 2)] for j in (2, 6, 12, 15)]
    ins = xs + xs[:5] + [taps[TAP_DCAT3], taps[TAP_DCAT2]]
    for i, (name, x) in enumerate(zip(HEADS, ins)):
        w = sd[name + ".0.weight"].to(dev).double()
        raw = taps[TAP_HEAD0 + i]
        r, kind = conv_ratio([nchw(x)], raw, [(w, None, 1, 0)], False, mode)
        yield name + ".conv", r, kind, float(x.abs().max())
        dst, off = HEAD_DST[i]
        c = w.shape[0]
        sl = taps[dst][..., off:off + c]
        r = gn_ratio(raw, sd[name + ".1.weight"].to(dev), sd[name + ".1.bias"].to(dev), HEAD_GROUPS[i], HEAD_UP[i], sl)
        yield name + ".gn_up_relu", r, "fp32", float(raw.abs().max())
    w6 = sd["fc_edge6.weight"].to(dev).double().flatten(1)
    r = smalln_ratio(taps[TAP_ECAT], w6, sd["fc_edge6.bias"].to(dev).double(), taps[TAP_ELOG], 5)
    yield "fc_edge6", r, "fp32", float(taps[TAP_ECAT].abs().max())
    w7 = sd["fc_dp7.3.weight"].to(dev).double().flatten(1)
    r = smalln_ratio(taps[TAP_DP7A], w7, -sd["mean_shift.running_mean"].to(dev).double(), taps[TAP_DLOG], 8)
    yield "fc_dp7.3+mean_shift", r, "fp32", float(taps[TAP_DP7A].abs().max())


def gn_fp32(raw, gam, bet, groups, up, hd, wd, dy=0.0, dmean=None):
    """gn_up_relu_kernel's arithmetic in torch-CPU fp32 (fp64 statistics) on raw NHWC -> NHWC; for the checker's own tests the
    bilinear row weight can be shifted by dy and group 0's mean scaled by (1 + dmean)"""
    x = nchw(raw).double()
    Bn, C, H, W = x.shape
    xg = x.reshape(Bn, groups, -1)
    mu = xg.mean(-1)
    var = (xg * xg).mean(-1) - mu * mu
    if dmean is not None:
        mu[:, 0] = mu[:, 0] * (1 + dmean)
    rstd = (1.0 / torch.sqrt(var + 1e-5)).float()
    cpg = C // groups
    m32, r32 = mu.float().repeat_interleave(cpg, 1)[..., None, None], rstd.repeat_interleave(cpg, 1)[..., None, None]
    v = (nchw(raw) - m32) * r32 * gam.view(1, -1, 1, 1) + bet.view(1, -1, 1, 1)
    if up > 1:
        Y = torch.arange(hd, dtype=torch.float32)
        X = torch.arange(wd, dtype=torch.float32)
        sy = ((Y + 0.5) / up - 0.5).clamp(min=0)
        sx = ((X + 0.5) / up - 0.5).clamp(min=0)
        y0, x0 = sy.long().clamp(max=H - 1), sx.long().clamp(max=W - 1)
        y1, x1 = (y0 + (y0 < H - 1).long()), (x0 + (x0 < W - 1).long())
        ly, lx = (sy - y0.float() + dy)[:, None], (sx - x0.float())[None, :]
        g = lambda yy, xx: v[:, :, yy][:, :, :, xx]
        v = (1 - ly) * ((1 - lx) * g(y0, x0) + lx * g(y0, x1)) + ly * ((1 - lx) * g(y1, x0) + lx * g(y1, x1))
    return F.relu(v[..., :hd, :wd]).permute(0, 2, 3, 1)


def cpu_taps(x, sd, kind):
    """Every tap of a forward as torch-CPU fp32 evaluates it (folded BN, as the plan stores it; GroupNorm statistics in fp64,
    as gn_partial_kernel keeps them), keyed by tap id, NHWC: the fp32 arithmetic the mode-0 bounds describe."""
    def nhwc(t):
        return t.permute(0, 2, 3, 1).contiguous()

    def conv(xi, conv_key, bn, st, pad, res=None, relu=True):
        w, b = fold(sd, conv_key, bn)
        y = F.conv2d(xi, w.float(), None if b is None else b.float(), stride=st, padding=pad)
        if res is not None:
            y = y + res
        return F.relu(y) if relu else y

    taps = {}
    y = conv(x, "resnet50.conv1.weight", "resnet50.bn1", 2, 3)
    taps[TAP_STEM] = nhwc(y)
    y = F.max_pool2d(y, 3, 2, 1)
    taps[TAP_POOL] = nhwc(y)
    for j, p, planes, st, first in blocks():
        t1 = conv(y, p + ".conv1.weight", p + ".bn1", 1, 0)
        t2 = conv(t1, p + ".conv2.weight", p + ".bn2", st, 1)
        res = conv(y, p + ".downsample.0.weight", p + ".downsample.1", st, 0, relu=False) if first else y
        y = conv(t2, p + ".conv3.weight", p + ".bn3", 1, 0, res=res)
        taps[block_tap(j, 0)], taps[block_tap(j, 1)], taps[block_tap(j, 2)] = nhwc(t1), nhwc(t2), nhwc(y)
    if kind == 0:
        return taps
    feats = [taps[TAP_POOL]] + [taps[block_tap(j, 2)] for j in (2, 6, 12, 15)]
    h2, w2 = feats[1].shape[1:3]
    h3, w3 = feats[2].shape[1:3]
    cat = {TAP_ECAT: [], TAP_DCAT2: [None, None, None], TAP_DCAT3: []}

    def head(i, xin, hd, wd):
        name = HEADS[i]
        raw = nhwc(F.conv2d(nchw(xin), sd[name + ".0.weight"]))
        taps[TAP_HEAD0 + i] = raw
        return gn_fp32(raw, sd[name + ".1.weight"], sd[name + ".1.bias"], HEAD_GROUPS[i], HEAD_UP[i], hd, wd)

    taps[TAP_ECAT] = torch.cat([head(i, feats[i], h2, w2) for i in range(5)], -1)
    taps[TAP_ELOG] = taps[TAP_ECAT] @ sd["fc_edge6.weight"].flatten(1).t() + sd["fc_edge6.bias"]
    d1, d2 = head(5, feats[0], h2, w2), head(6, feats[1], h2, w2)
    taps[TAP_DCAT3] = torch.cat([head(7, feats[2], h3, w3), head(8, feats[3], h3, w3), head(9, feats[4], h3, w3)], -1)
    taps[TAP_DCAT2] = torch.cat([d1, d2, head(10, taps[TAP_DCAT3], h2, w2)], -1)
    taps[TAP_DP7A] = head(11, taps[TAP_DCAT2], h2, w2)
    taps[TAP_DLOG] = taps[TAP_DP7A] @ sd["fc_dp7.3.weight"].flatten(1).t() - sd["mean_shift.running_mean"]
    return taps
