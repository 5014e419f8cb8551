"""Parameter containers whose ``state_dict()`` keys equal the reference's.

The reference checkpoints (`sess/res50_cam.pth.pth`, `sess/res50_irn.pth`) carry every
tensor under several alias keys because the same sub-modules are registered under
`resnet50.*`, `stageN.*` and `backbone.*` (SURVEY.md D10; net/resnet50_cam.py:12-23,
net/resnet50_irn.py:14-97).  `load_state_dict(strict=True)` therefore needs the same module
tree.  The modules here are parameter HOLDERS only: nothing calls their torch `forward`;
the arithmetic runs in irn_b200/csrc through the C ABI.
"""
import torch
import torch.nn as nn

# (planes, blocks, stride) for layer1..4 under the reference's strides=(2,2,2,1)
TRUNK = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 1))


def _conv(cin, cout, k, bias=False):
    return nn.Conv2d(cin, cout, k, bias=bias)


class _Block(nn.Module):
    def __init__(self, cin, planes, stride, project):
        super().__init__()
        self.conv1, self.bn1 = _conv(cin, planes, 1), nn.BatchNorm2d(planes)
        self.conv2, self.bn2 = _conv(planes, planes, 3), nn.BatchNorm2d(planes)
        self.conv3, self.bn3 = _conv(planes, planes * 4, 1), nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU()
        self.downsample = (nn.Sequential(_conv(cin, planes * 4, 1), nn.BatchNorm2d(planes * 4))
                           if project else None)
        self.stride = stride


class _Trunk(nn.Module):
    """ResNet-50 parameter tree (names as net/resnet50.py:59-72)."""

    def __init__(self):
        super().__init__()
        self.conv1, self.bn1 = _conv(3, 64, 7), nn.BatchNorm2d(64)
        self.relu, self.maxpool = nn.ReLU(), nn.MaxPool2d(3, 2, 1)
        cin = 64
        for i, (planes, blocks, stride) in enumerate(TRUNK, start=1):
            seq = [_Block(cin, planes, stride, True)]
            cin = planes * 4
            seq += [_Block(cin, planes, 1, False) for _ in range(blocks - 1)]
            setattr(self, "layer%d" % i, nn.Sequential(*seq))


MAX_CLASSES = 128   # IRN_CAM_MAX_CLASSES of include/irn_b200.h


class CamParams(nn.Module):
    """Key-compatible with net/resnet50_cam.py:9-23 (Net / CAM).  The classifier has `n_classes` rows: 20 for PASCAL VOC (the
    reference), 80 for MS COCO."""

    def __init__(self, n_classes=20):
        super().__init__()
        if not 1 <= int(n_classes) <= MAX_CLASSES:
            raise ValueError("a CAM network has 1..%d classes, got %s" % (MAX_CLASSES, n_classes))
        t = self.resnet50 = _Trunk()
        self.stage1 = nn.Sequential(t.conv1, t.bn1, t.relu, t.maxpool, t.layer1)
        self.stage2 = nn.Sequential(t.layer2)
        self.stage3 = nn.Sequential(t.layer3)
        self.stage4 = nn.Sequential(t.layer4)
        self.classifier = _conv(2048, int(n_classes), 1)
        self.backbone = nn.ModuleList([self.stage1, self.stage2, self.stage3, self.stage4])
        self.newly_added = nn.ModuleList([self.classifier])


class _MeanShift(nn.Module):
    def __init__(self, n):
        super().__init__()
        self.register_buffer("running_mean", torch.zeros(n))


# head name -> (cin, cout, groups, upsample factor)   (net/resnet50_irn.py:23-93)
EDGE_HEADS = (("fc_edge1", 64, 32, 4, 1), ("fc_edge2", 256, 32, 4, 1), ("fc_edge3", 512, 32, 4, 2),
              ("fc_edge4", 1024, 32, 4, 4), ("fc_edge5", 2048, 32, 4, 4))
DP_HEADS = (("fc_dp1", 64, 64, 8, 1), ("fc_dp2", 256, 128, 16, 1), ("fc_dp3", 512, 256, 16, 1),
            ("fc_dp4", 1024, 256, 16, 2), ("fc_dp5", 2048, 256, 16, 2), ("fc_dp6", 768, 256, 16, 2),
            ("fc_dp7", 448, 256, 16, 1))


def _head(cin, cout, groups, up):
    mods = [_conv(cin, cout, 1), nn.GroupNorm(groups, cout)]
    if up > 1:
        mods.append(nn.Upsample(scale_factor=up, mode="bilinear", align_corners=False))
    mods.append(nn.ReLU())
    return mods


class IrnParams(nn.Module):
    """Key-compatible with net/resnet50_irn.py:9-97 (Net / EdgeDisplacement)."""

    def __init__(self):
        super().__init__()
        t = self.resnet50 = _Trunk()
        self.stage1 = nn.Sequential(t.conv1, t.bn1, t.relu, t.maxpool)
        self.stage2 = nn.Sequential(t.layer1)
        self.stage3 = nn.Sequential(t.layer2)
        self.stage4 = nn.Sequential(t.layer3)
        self.stage5 = nn.Sequential(t.layer4)
        self.mean_shift = _MeanShift(2)
        for name, cin, cout, g, up in EDGE_HEADS:
            setattr(self, name, nn.Sequential(*_head(cin, cout, g, up)))
        self.fc_edge6 = _conv(160, 1, 1, bias=True)
        for name, cin, cout, g, up in DP_HEADS:
            mods = _head(cin, cout, g, up)
            if name == "fc_dp7":
                mods += [_conv(256, 2, 1), self.mean_shift]
            setattr(self, name, nn.Sequential(*mods))
        self.backbone = nn.ModuleList([self.stage1, self.stage2, self.stage3, self.stage4, self.stage5])
        self.edge_layers = nn.ModuleList([getattr(self, n[0]) for n in EDGE_HEADS] + [self.fc_edge6])
        self.dp_layers = nn.ModuleList([getattr(self, n[0]) for n in DP_HEADS])
