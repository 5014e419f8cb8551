"""CPU checks of the per-layer checker (tests/layer_check.py), the tap shapes and the trained-like checkpoint.

The checker must accept torch-CPU fp32 (the arithmetic its mode-0 bound describes) and reject small, systematic errors:
a wrong bias on a small-valued channel next to large ones, one bilinear weight off by 2^-12, one GroupNorm group's mean
off by 2^-16 of its magnitude."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import layer_check as lc
from irn_b200 import synth
from irn_b200.cam import CAM, tap_shape
from irn_b200.irn import EdgeDisplacement
from oracle import nets


def _input(P, H, W, seed=5):
    xs = []
    for p in range(P):
        xi = synth.normalize_image(synth.image(seed + p, H, W))
        xs += [xi, xi[..., ::-1].copy()]
    return torch.from_numpy(np.stack(xs))


@pytest.fixture(scope="module")
def irn_case():
    sd = lc.hostile_irn_state_dict()
    x = _input(1, 64, 64)
    return sd, x, lc.cpu_taps(x, sd, 1)


@pytest.mark.parametrize("ckpt", ["synth", "trained_like"])
def test_checker_accepts_fp32(ckpt):
    sd = synth.cam_state_dict() if ckpt == "synth" else lc.hostile_cam_state_dict()
    x = _input(1, 48, 80)
    taps = lc.cpu_taps(x, sd, 0)
    worst = max(r for _, r, _, _ in lc.trunk_layers(sd, taps, x, 0))
    assert worst <= 1.0
    assert worst > 1e-3, "the mode-0 bound is too loose to catch anything (worst ratio %g)" % worst


def test_checker_accepts_fp32_heads(irn_case):
    sd, x, taps = irn_case
    rows = list(lc.irn_head_layers(sd, taps, 0))
    assert len(rows) == 26
    for name, r, _, _ in rows:
        assert r <= 1.0, name


def test_checker_rejects_small_channel_bias():
    """One small-valued channel's bias off by 4 times its own bound: per element that is rejected, while the error is far
    below 1e-5 of the tensor's max (what a max-relative check would allow): the trained-like checkpoint's channels span
    binades."""
    sd = lc.hostile_cam_state_dict()
    x = _input(1, 48, 80)
    taps = lc.cpu_taps(x, sd, 0)
    p = "resnet50.layer1.0"
    t1 = taps[lc.block_tap(0, 0)]
    w, b = lc.fold(sd, p + ".conv1.weight", p + ".bn1")
    A = F.conv2d(lc.nchw(taps[lc.TAP_POOL]).double().abs(), w.abs(), b.abs())
    live = (t1 > 0).all(dim=(0, 1, 2))
    c = int(torch.where(live, A.amax(dim=(0, 2, 3)), torch.full_like(A[0, :, 0, 0], np.inf)).argmin())
    bound = lc.eps_for("simt", 64, 0) * float(A[:, c].amax())
    y = t1.clone()
    y[..., c] += 4 * bound
    assert 4 * bound < 1e-5 * float(t1.abs().max())
    r, _ = lc.conv_ratio([lc.nchw(taps[lc.TAP_POOL])], y, [(w, b, 1, 0)], True, 0)
    assert r > 1.0
    r0, _ = lc.conv_ratio([lc.nchw(taps[lc.TAP_POOL])], t1, [(w, b, 1, 0)], True, 0)
    assert r0 <= 1.0


def test_checker_gn_fp32_and_perturbations(irn_case):
    sd, x, taps = irn_case
    i = 3   # fc_edge4: x4 upsample, group 0 has a mean far above its std
    name = lc.HEADS[i]
    raw = taps[lc.TAP_HEAD0 + i]
    gam, bet = sd[name + ".1.weight"], sd[name + ".1.bias"]
    dst, off = lc.HEAD_DST[i]
    hd, wd = taps[dst].shape[1:3]
    xg = lc.nchw(raw).double().reshape(raw.shape[0], 4, -1)
    assert float((xg[:, 0].mean(-1).abs() / xg[:, 0].std(-1)).min()) > 5, "group 0's mean should dwarf its std"
    args = (raw, gam, bet, 4, 4, hd, wd)
    assert lc.gn_ratio(raw, gam, bet, 4, 4, lc.gn_fp32(*args)) <= 1.0
    assert lc.gn_ratio(raw, gam, bet, 4, 4, lc.gn_fp32(*args, dy=2.0 ** -12)) > 1.0
    assert lc.gn_ratio(raw, gam, bet, 4, 4, lc.gn_fp32(*args, dmean=2.0 ** -16)) > 1.0
    # torch's own fp32 GroupNorm forms the variance in fp32: on that group it is rejected too
    z = F.interpolate(F.group_norm(lc.nchw(raw), 4, gam, bet, eps=1e-5), scale_factor=4, mode="bilinear", align_corners=False)
    assert lc.gn_ratio(raw, gam, bet, 4, 4, F.relu(z[..., :hd, :wd]).permute(0, 2, 3, 1)) > 1.0


def test_tap_shapes_match_oracle(built_lib, irn_case):
    sd, x, taps = irn_case
    for i in range(lc.TAP_COUNT):
        assert tap_shape(1, i, x.shape[0], crop_size=64) == tuple(taps[i].shape), i
    cam_taps = lc.cpu_taps(_input(2, 40, 72), synth.cam_state_dict(), 0)
    for i in range(lc.TAP_BLOCK0 + 48):
        assert tap_shape(0, i, 4, 40, 72) == tuple(cam_taps[i].shape), i
    assert tap_shape(0, lc.TAP_CAM_CLS, 4, 40, 72) == (4, 3, 5, 64)
    with pytest.raises(Exception):
        tap_shape(0, lc.TAP_CAM_CLS + 1, 4, 40, 72)


def test_trained_like_checkpoint():
    """Loads (CAM strictly), has the stated statistics, and keeps every f16x3 layer input below 65504 with a CAM that is
    not degenerate (the oracle at 128x160)."""
    cam_sd, irn_sd = lc.hostile_cam_state_dict(), lc.hostile_irn_state_dict()
    CAM().load_state_dict(cam_sd, strict=True)
    EdgeDisplacement().load_state_dict(irn_sd, strict=False)
    g = torch.cat([v for k, v in cam_sd.items() if k.startswith("resnet50.") and k.endswith("bn2.weight")])
    assert 0.02 < float((g == 0).float().mean()) < 0.1 and 0.05 < float((g < 0).float().mean()) < 0.15
    v = torch.cat([v for k, v in cam_sd.items() if k.startswith("resnet50.") and k.endswith("running_var")])
    s = (torch.cat([v for k, v in cam_sd.items() if k.startswith("resnet50.") and k.endswith("bn2.weight")]).abs() /
         torch.cat([v for k, v in cam_sd.items() if k.startswith("resnet50.") and k.endswith("bn2.running_var")]).sqrt())
    s = s[s > 0]
    assert float(torch.log2(s.max() / s.min())) > 10 and float(v.min()) < 1e-3 and float(v.max()) > 10
    x = _input(1, 128, 160)
    taps = lc.cpu_taps(x, cam_sd, 0)
    for j, p, *_ in lc.blocks():
        for which in range(3):
            assert float(taps[lc.block_tap(j, which)].abs().max()) < lc.F16_MAX, "%s tap %d" % (p, which)
    cam = nets.cam_forward(x, cam_sd)
    assert float((cam > 0).float().mean()) > 0.1 and float(cam.max()) > 0
    itaps = lc.cpu_taps(_input(1, 64, 64), irn_sd, 1)
    assert all(float(t.abs().max()) < lc.F16_MAX for t in itaps.values())
