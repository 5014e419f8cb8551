"""Seeded synthetic checkpoints, images and kernel-level inputs (SURVEY.md section 8(d)).

There is no network and no VOC data: weights are random-initialised in the reference's
checkpoint format (same keys, so the reference's own `load_state_dict(strict=True)` accepts
them), images are VOC-shaped uint8 [H,W,3].  Pure numpy/torch-CPU; used by tests, bench.py
and tests/golden/make_golden.py so that every party sees identical data.
"""
import numpy as np
import torch

from . import _params


def _fill_trunk(trunk, g):
    for name, m in trunk.named_modules():
        if isinstance(m, torch.nn.Conv2d):
            fan_in = m.in_channels * m.kernel_size[0] * m.kernel_size[1]
            m.weight.data = torch.randn(m.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5
        elif isinstance(m, torch.nn.BatchNorm2d):
            c = m.num_features
            last = name.endswith("bn3") or name.endswith("downsample.1")
            # bn3 / projection gains < 1 keep the residual stream bounded over 16 blocks
            m.weight.data = (0.5 if last else 1.0) * (1 + 0.1 * torch.randn(c, generator=g))
            m.bias.data = 0.05 * torch.randn(c, generator=g)
            m.running_mean.data = 0.1 * torch.randn(c, generator=g)
            m.running_var.data = 1 + 0.2 * torch.rand(c, generator=g)


def cam_state_dict(seed=0, n_classes=20):
    """Reference-format state dict for net.resnet50_cam.CAM (956 keys with aliases), with an `n_classes`-row classifier."""
    g = torch.Generator().manual_seed(seed)
    m = _params.CamParams(n_classes)
    _fill_trunk(m.resnet50, g)
    m.classifier.weight.data = 0.01 * torch.randn(m.classifier.weight.shape, generator=g)
    return {k: v.clone() for k, v in m.state_dict().items()}


def irn_state_dict(seed=1, edge_gain=6.0):
    """Reference-format state dict for net.resnet50_irn.EdgeDisplacement.

    `edge_gain` scales fc_edge6 so that the edge logits are spread enough for sigmoid(edge)
    to be bimodal-ish; with torch-default init every edge sits near 0.6 and the random walk
    degenerates to the identity (SURVEY.md section 8(d))."""
    g = torch.Generator().manual_seed(seed)
    m = _params.IrnParams()
    _fill_trunk(m.resnet50, g)
    for name, mod in m.named_modules():
        if name.startswith("fc_") and isinstance(mod, torch.nn.Conv2d):
            fan_in = mod.in_channels
            mod.weight.data = torch.randn(mod.weight.shape, generator=g) * (1.0 / fan_in) ** 0.5
        elif name.startswith("fc_") and isinstance(mod, torch.nn.GroupNorm):
            c = mod.num_channels
            mod.weight.data = 1 + 0.1 * torch.randn(c, generator=g)
            mod.bias.data = 0.1 * torch.randn(c, generator=g)
    m.fc_edge6.weight.data *= edge_gain
    m.fc_edge6.bias.data = torch.tensor([-1.0])
    m.mean_shift.running_mean.data = torch.tensor([0.1, -0.05])
    return {k: v.clone() for k, v in m.state_dict().items()}


def image(index, H=512, W=512):
    """VOC-shaped synthetic uint8 image: soft coloured ellipses over a low-frequency
    background plus N(0,8) noise (white noise alone gives degenerate CAMs)."""
    rng = np.random.default_rng(1234 + int(index))
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    img = np.empty((H, W, 3), np.float32)
    for c in range(3):
        fy, fx = rng.uniform(0.5, 2.0, 2)
        ph = rng.uniform(0, 6.28, 2)
        img[..., c] = 110 + 40 * np.sin(fy * yy / H * 6.28 + ph[0]) * np.cos(fx * xx / W * 6.28 + ph[1])
    for _ in range(int(rng.integers(3, 7))):
        cy, cx = rng.uniform(0.15, 0.85) * H, rng.uniform(0.15, 0.85) * W
        ry, rx = rng.uniform(0.06, 0.3) * H, rng.uniform(0.06, 0.3) * W
        col = rng.uniform(0, 255, 3).astype(np.float32)
        with np.errstate(over="ignore"):   # exp overflow -> inf -> m = 0 exactly, intended
            m = 1.0 / (1.0 + np.exp(8.0 * (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 - 1.0)))
        img = img * (1 - m[..., None]) + col * m[..., None]
    img += rng.normal(0, 8, img.shape).astype(np.float32)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def label(index, n_present=None, n_classes=20):
    """Multi-hot fp32[n_classes] with 1..3 classes (mean ~1.5, like voc12/cls_labels.npy)."""
    rng = np.random.default_rng(977 + int(index))
    k = n_present if n_present is not None else int(rng.choice([1, 2, 3], p=[0.62, 0.30, 0.08]))
    lab = np.zeros(n_classes, np.float32)
    lab[rng.choice(n_classes, size=k, replace=False)] = 1
    return lab


def _blur(a, k):
    ker = np.ones(k, np.float32) / k
    a = np.apply_along_axis(lambda v: np.convolve(v, ker, mode="same"), 0, a)
    return np.apply_along_axis(lambda v: np.convolve(v, ker, mode="same"), 1, a)


def edge_map(h, w, kind="bimodal", seed=0):
    """Kernel-level edge inputs in (0,1), fp32 [1,h,w]: the four distributions of
    SURVEY.md App. B."""
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        e = rng.random((h, w))
    elif kind == "sigmoid4":
        e = 1 / (1 + np.exp(-4 * rng.standard_normal((h, w))))
    elif kind == "low":
        e = 0.1 * rng.random((h, w))
    else:
        z = _blur(rng.standard_normal((h, w)).astype(np.float32), 9)
        z = z / (z.std() + 1e-6)
        with np.errstate(over="ignore"):
            e = 1 / (1 + np.exp(30 * (np.abs(z) - 0.12)))   # thin ridges where |z| is small
    return e.astype(np.float32)[None]


def seeds(C, h, w, seed=0):
    return np.random.default_rng(1000 + seed).random((C, h, w)).astype(np.float32)


def displacement(h, w, n_attractors=3, seed=0):
    """dp fp32 [2,h,w] = 0.2*(nearest attractor - coord) + N(0,0.05)."""
    rng = np.random.default_rng(500 + seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    att = np.stack([rng.uniform(0.15, 0.85, n_attractors) * h, rng.uniform(0.15, 0.85, n_attractors) * w], 1)
    d = np.stack([att[:, 0][:, None, None] - yy, att[:, 1][:, None, None] - xx], 1)
    near = np.argmin((d ** 2).sum(1), 0)
    dp = np.take_along_axis(d, near[None, None].repeat(2, 1), 0)[0] * 0.2
    return (dp + rng.normal(0, 0.05, (2, h, w))).astype(np.float32)


def normalize_image(img_u8):
    """TorchvisionNormalize + HWC->CHW (voc12/dataloader.py:65-78): fp32 [3,H,W]."""
    mean = (0.485, 0.456, 0.406)
    std = (0.229, 0.224, 0.225)
    a = np.asarray(img_u8)
    out = np.empty(a.shape, np.float32)
    for c in range(3):
        out[..., c] = (a[..., c] / 255. - mean[c]) / std[c]
    return np.ascontiguousarray(out.transpose(2, 0, 1))


def cam_planes_u8(K, H, W, seed=0):
    """K structured CAM-like planes quantised to uint8 (a few Gaussian blobs each, peak 255): the stored CAMs of the
    cam_to_ir_label fixtures are `u8 / 255` in float32, so the exact inputs travel as compressible bytes."""
    rs = np.random.RandomState(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.zeros((K, H, W), np.uint8)
    for k in range(K):
        a = np.zeros((H, W))
        for _ in range(rs.randint(1, 4)):
            cy, cx = rs.uniform(0, H), rs.uniform(0, W)
            sy, sx = rs.uniform(0.08, 0.3) * H, rs.uniform(0.08, 0.3) * W
            a += rs.uniform(0.3, 1.0) * np.exp(-0.5 * (((y - cy) / sy) ** 2 + ((x - cx) / sx) ** 2))
        out[k] = np.round(255 * a / a.max()).astype(np.uint8)
    return out


def u8_to_cam(u8):
    return np.asarray(u8).astype(np.float32) / np.float32(255)
