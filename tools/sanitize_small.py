"""Small-shape tour of every hand-written kernel family, meant to run under compute-sanitizer (memcheck / racecheck /
initcheck): fused cluster walk at every cluster size 1..16, the per-step walk, the wgmma convolution kernels (3xTF32 and
f16x3, every N tile, the tensor-core stems, the fused conv3 + projection shortcut), labels, CAM merge, instance kernels, input
pyramids.
    compute-sanitizer --tool memcheck python tools/sanitize_small.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from irn_b200 import cam_ops, indexing, instance, preprocess, synth
from irn_b200.ops import Conv2d, ShortcutConv, Stem

dev = torch.device("cuda:0")
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)

# random walk: cluster sizes 1, 2, 4, 8, 16 (8 rows per CTA), fused and per-step kernels, two channels
for h, w in [(8, 40), (16, 33), (30, 64), (60, 50), (128, 128)]:
    e, x = synth.edge_map(h, w, "bimodal", h), synth.seeds(2, h, w, w)
    for variant in (4, 2, 1):
        indexing.random_walk_batch(t(x), t(e), [0, 2], n_iter=3, variant=variant)
    torch.cuda.synchronize()
    print("walk", h, w, "ok", flush=True)

# convolutions: (cin, cout, k, stride, H, W, residual) -> every wgmma kernel configuration once
for cin, cout, k, s, H, W, res in [(64, 64, 3, 1, 20, 24, False), (64, 256, 1, 1, 20, 24, True), (256, 64, 1, 1, 20, 24, False),
                                   (128, 128, 3, 2, 24, 24, False), (256, 256, 3, 1, 16, 16, False), (1024, 256, 1, 1, 16, 16, False),
                                   (512, 1024, 1, 2, 16, 16, False)]:
    w_ = (torch.randn(cout, cin, k, k) * 0.05).numpy()
    conv = Conv2d(w_, None, s, k // 2)
    x = torch.randn(2, H, W, cin).to(dev)            # host-generated + H2D copy: initcheck does not see PyTorch's own generator kernels' writes
    Ho = (H + 2 * (k // 2) - k) // s + 1
    Wo = (W + 2 * (k // 2) - k) // s + 1
    r = torch.randn(2, Ho, Wo, cout).to(dev) if res else None
    for mode in (1, 2):
        conv(x, r, relu=True, mode=mode)
    torch.cuda.synchronize()
    print("conv", cin, cout, k, s, "ok", flush=True)
bn = lambda n: [np.ones(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32), np.ones(n, np.float32)]
stem = Stem((torch.randn(64, 3, 7, 7) * 0.05).numpy(), bn(64))
for mode in (1, 2):
    stem(torch.randn(2, 3, 30, 41).to(dev), 48, 48, mode=mode)   # crop padding: H, W < Hin, Win
sc = ShortcutConv((torch.randn(512, 128) * 0.05).numpy(), bn(512), (torch.randn(512, 256) * 0.05).numpy(), bn(512), 2)
sc(torch.randn(2, 7, 9, 128).to(dev), torch.randn(2, 13, 17, 256).to(dev))
torch.cuda.synchronize()
print("stem, fused shortcut ok", flush=True)

# labels, merge, instance kernels, pyramids
rw = torch.rand(3, 20, 24).to(dev)
indexing.rw_labels(rw, [1, 4, 7], (78, 95), want_index=True, want_scores=True)
cams = [torch.rand(20, s_, s_ + 1).to(dev) for s_ in (5, 3, 8, 10)]
lab = np.zeros(20, np.float32); lab[[2, 9]] = 1
cam_ops.merge_cams(cams, (78, 95), lab)
dp = t(synth.displacement(20, 24, 3, 1))
cen = instance.find_centroids_with_refinement(dp, iterations=20)
inst, n = instance.cluster_centroids(cen, dp)
seeds = instance.separate_score_by_mask(torch.rand(2, 20, 24).to(dev), inst, n)
_, idx, sc = indexing.rw_labels(seeds.reshape(-1, 20, 24), None, (78, 95), want_index=True, want_scores=True)
instance.detect_instance(sc, idx, np.repeat([1, 2], n), 10)
preprocess.msf_batch(t(synth.image(1, 37, 50)[None]), (1.0, 0.5, 1.5))
torch.cuda.synchronize()
print("misc ok", flush=True)
