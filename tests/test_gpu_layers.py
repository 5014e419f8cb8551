"""Every CAM and IRNet layer against float64 on its own input, per element, with condition-aware bounds
(tests/layer_check.py derives them), on the seeded synthetic checkpoint and on a trained-like one.

The trained-like checkpoint (layer_check.hostile_*_state_dict) has BatchNorm statistics like a trained ResNet-50's:
~5 % dead channels (gamma = 0), ~10 % negative gamma, |gamma| log-uniform over 8 binades, running_var log-uniform over
1e-4 .. 1e2 (folded scales over 20 binades), running_mean of a few standard deviations (bias-dominated channels whose fold
cancels), GroupNorm heads with zero / negative gamma and a group per head whose mean dwarfs its std.  Stated precondition:
every f16x3 layer input stays below 65504 in magnitude (the activation split saturates there); a violation fails naming
the layer.

Inputs: the four pyramid scales of one 512x512 image (CAM inputs 256..1024, the benchmark's shapes), a 2-pair batch of a
375x500 image at scale 1.5 (563x750: odd extents, ragged tiles); IRNet: P = 2 pairs of 375x500 and P = 1 of 512x512 on the
512 canvas.  Each layer's worst |y - y64| / bound goes to conftest.record."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import layer_check as lc
from conftest import record
from irn_b200 import synth
from irn_b200.cam import CAM, tap_shape
from irn_b200.irn import EdgeDisplacement
from oracle import nets
from oracle import resize as oracle_resize

pytestmark = pytest.mark.gpu

CKPTS = ["synth", "trained_like"]
MODES = [0, 1, 2]


@pytest.fixture(autouse=True)
def fp64_references_without_tf32():
    """The fp64 references run in fp64, and torch's fp32 helpers here must not round through TF32; the switches are restored
    afterwards so no other test sees them changed."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.fixture(scope="module")
def state_dicts():
    return {"synth": (synth.cam_state_dict(), synth.irn_state_dict()),
            "trained_like": (lc.hostile_cam_state_dict(), lc.hostile_irn_state_dict())}


def _cam_inputs():
    pyr = oracle_resize.msf_preprocess(synth.image(0, 512, 512), (0.5, 1.0, 1.5, 2.0))
    out = {"512@%s" % s: p for s, p in zip((0.5, 1.0, 1.5, 2.0), pyr)}
    a = oracle_resize.msf_preprocess(synth.image(1, 375, 500), (1.5,))[0]
    b = oracle_resize.msf_preprocess(synth.image(2, 375, 500), (1.5,))[0]
    out["375x500@1.5x2"] = np.concatenate([a, b])
    return out


CAM_INPUTS = _cam_inputs()


def _forward_with_taps(model, kind, ids, x, dev, crop=0):
    B, _, H, W = x.shape
    taps = {}
    for i in ids:
        taps[i] = torch.full(tap_shape(kind, i, B, H, W, crop), float("nan"), device=dev)
        model.set_tap(i, taps[i])
    try:
        out = model.forward_batch(x)
        torch.cuda.synchronize()
    finally:
        for i in ids:
            model.set_tap(i, None, device=dev)
    return out, taps


def _check(name, rows, **ctx):
    bad = []
    for layer, r, kind, xmax in rows:
        record(name, layer=layer, arith=kind, ratio=r, **ctx)
        if kind == "f16":
            assert xmax < lc.F16_MAX, "precondition: %s input reaches %g >= 65504, the f16x3 split saturates" % (layer, xmax)
        if not r <= 1.0:
            bad.append("%s (%s): %.3g" % (layer, kind, r))
    assert not bad, "layers over their derived bound: " + ", ".join(bad)


@pytest.mark.parametrize("inp", list(CAM_INPUTS))
@pytest.mark.parametrize("ckpt", CKPTS)
@pytest.mark.parametrize("mode", MODES)
def test_cam_layers(cuda_dev, state_dicts, mode, ckpt, inp):
    sd = state_dicts[ckpt][0]
    m = CAM()
    m.load_state_dict(sd, strict=True)
    m.set_conv_mode(mode)
    x = torch.from_numpy(CAM_INPUTS[inp]).to(cuda_dev)
    ids = list(range(lc.TAP_BLOCK0 + 48)) + ([lc.TAP_CAM_CLS] if mode else [])
    cam, taps = _forward_with_taps(m, 0, ids, x, cuda_dev)
    ctx = dict(mode=mode, ckpt=ckpt, input=inp)
    assert lc.maxpool_exact(taps), "max pool differs from F.max_pool2d of the stem output"
    rows = list(lc.trunk_layers(sd, taps, x, mode))
    feat = taps[lc.block_tap(15, 2)]
    w = sd["classifier.weight"].to(cuda_dev).double()
    if mode:
        tmp = taps[lc.TAP_CAM_CLS]
        wp = torch.cat([w, w.new_zeros(44, 2048, 1, 1)])
        r, kind = lc.conv_ratio([lc.nchw(feat)], tmp, [(wp, None, 1, 0)], True, mode)
        rows.append(("classifier", r, kind, float(feat.abs().max())))
        t = tmp[..., :20]
        ref = (t[0::2] + t[1::2].flip(2)).permute(0, 3, 1, 2)
        assert torch.equal(cam, ref), "cam_flip_add differs from the fp32 sum of the classifier tap"
    else:   # cam_head_kernel: per sample a 2048-term dot product over 32 lanes (64 FMAs + 5 adds), ReLU, one add
        f64 = feat.double()
        z = F.relu(f64 @ w.flatten(1).t())
        A = f64.abs() @ w.flatten(1).abs().t()
        ref = (z[0::2] + z[1::2].flip(2)).permute(0, 3, 1, 2)
        bound = lc.gamma(64 + 5 + 1) * (A[0::2] + A[1::2].flip(2)).permute(0, 3, 1, 2)
        rows.append(("cam_head", lc._ratio((cam.double() - ref).abs(), bound), "simt", float(feat.abs().max())))
    _check("gpu_layers_cam", rows, **ctx)
    if ckpt == "trained_like":   # end to end against a pure fp64 oracle run (no reference fixture exists for this checkpoint)
        sd64 = {k: v.to(cuda_dev).double() for k, v in sd.items()}
        with torch.no_grad():
            err = 0.0
            for p in range(x.shape[0] // 2):
                ref = nets.cam_forward(x[2 * p:2 * p + 2].double(), sd64)
                err = max(err, float((cam[p].double() - ref).abs().max() / ref.abs().max()))
        record("gpu_layers_cam_e2e_fp64", normalised_err=err, **ctx)


IRN_INPUTS = {"2x375x500": (2, 375, 500), "1x512x512": (1, 512, 512)}


@pytest.mark.parametrize("inp", list(IRN_INPUTS))
@pytest.mark.parametrize("ckpt", CKPTS)
@pytest.mark.parametrize("mode", MODES)
def test_irn_layers(cuda_dev, state_dicts, mode, ckpt, inp):
    sd = state_dicts[ckpt][1]
    m = EdgeDisplacement()
    m.load_state_dict(sd, strict=False)
    m.set_conv_mode(mode)
    P, H, W = IRN_INPUTS[inp]
    xs = []
    for p in range(P):
        xi = synth.normalize_image(synth.image(10 + p, H, W))
        xs += [xi, xi[..., ::-1].copy()]
    x = torch.from_numpy(np.stack(xs)).to(cuda_dev)
    crop = 512
    (edge, dp), taps = _forward_with_taps(m, 1, list(range(lc.TAP_COUNT)), x, cuda_dev, crop)
    ctx = dict(mode=mode, ckpt=ckpt, input=inp)
    assert lc.maxpool_exact(taps), "max pool differs from F.max_pool2d of the stem output"
    x_in = F.pad(x, [0, crop - W, 0, crop - H])
    rows = list(lc.trunk_layers(sd, taps, x_in, mode)) + list(lc.irn_head_layers(sd, taps, mode))
    fh, fw = (H - 1) // 4 + 1, (W - 1) // 4 + 1
    rows.append(("edge_tail", lc.edge_tail_ratio(taps[lc.TAP_ELOG], edge, P, fh, fw), "fp32", 0.0))
    assert torch.equal(dp, taps[lc.TAP_DLOG][0::2, :fh, :fw].permute(0, 3, 1, 2)), "dp differs from the dp logits of sample 2p"
    _check("gpu_layers_irn", rows, **ctx)
    if ckpt == "trained_like":
        sd64 = {k: v.to(cuda_dev).double() for k, v in sd.items()}
        with torch.no_grad():
            ee = de = 0.0
            for p in range(P):
                e64, d64 = nets.edge_displacement(x[2 * p:2 * p + 2].double(), sd64, crop)
                ee = max(ee, float((edge[p].double() - e64).abs().max()))
                de = max(de, float((dp[p].double() - d64).abs().max() / d64.abs().max()))
        record("gpu_layers_irn_e2e_fp64", edge_abs_err=ee, dp_normalised_err=de, **ctx)


def test_taps_change_nothing(cuda_dev, state_dicts):
    """A forward with every tap set launches the same kernels and returns the same bits as one without."""
    from irn_b200 import _lib
    m = EdgeDisplacement()
    m.load_state_dict(state_dicts["synth"][1], strict=False)
    x = torch.from_numpy(CAM_INPUTS["512@0.5"]).to(cuda_dev)
    e0, d0 = m.forward_batch(x)
    n0 = _lib.lib().irn_total_launch_count()
    e0, d0 = m.forward_batch(x)
    n1 = _lib.lib().irn_total_launch_count()
    (e1, d1), _ = _forward_with_taps(m, 1, list(range(lc.TAP_COUNT)), x, cuda_dev, 512)
    n2 = _lib.lib().irn_total_launch_count()
    assert n2 - n1 == n1 - n0
    assert torch.equal(e0, e1) and torch.equal(d0, d1)
