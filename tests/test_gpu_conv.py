"""The convolution kernels (SIMT fp32 and wgmma 3xTF32) against a plain torch fp32 reference of the same
op (F.conv2d + batch_norm on the GPU with TF32 disabled)."""
import pytest
import torch
import torch.nn.functional as F

from irn_b200.ops import Conv2d

pytestmark = pytest.mark.gpu

CASES = [  # cin, cout, k, stride, pad, B, H, W
    (64, 256, 1, 1, 0, 2, 40, 48),
    (64, 64, 3, 1, 1, 2, 37, 53),      # ragged tiles
    (64, 64, 3, 1, 1, 4, 128, 160),    # 640 tiles, 18 k-blocks each
    (256, 64, 1, 1, 0, 4, 96, 128),    # 8 k-blocks per tile: ring wrap-around
    (64, 256, 1, 1, 0, 4, 96, 128),    # 768 tiles
    (128, 128, 3, 2, 1, 2, 64, 64),
    (256, 512, 1, 2, 0, 2, 33, 47),
    (512, 128, 1, 1, 0, 3, 16, 16),
    (512, 512, 3, 1, 1, 2, 20, 24),    # K = 4608: 144 k-blocks
    (1024, 256, 1, 1, 0, 2, 33, 17),
    (2048, 512, 1, 1, 0, 1, 16, 16),
    (3, 64, 7, 2, 3, 2, 64, 80),       # stem: SIMT only
    (2048, 32, 1, 1, 0, 2, 8, 8),      # edge head: SIMT only
    (256, 128, 3, 1, 1, 2, 19, 27, "nobn"),   # no bias: the IRNet head / classifier epilogue
]


def _with_relu(cases):
    """Every case with ReLU on (the id it always had) and off (suffix -norelu): with ReLU on, outputs where both the kernel
    and the reference are negative clamp to 0 and are never compared."""
    return [pytest.param(c, relu, id="x".join(map(str, c)) + ("" if relu else "-norelu")) for c in cases for relu in (True, False)]


@pytest.mark.parametrize("case,relu", _with_relu(CASES))
def test_conv_vs_torch(cuda_dev, case, relu):
    cin, cout, k, stride, pad, B, H, W, *opt = case
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(cin * 7 + cout + k)
    w = torch.randn((cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5
    bn = [1 + 0.1 * torch.randn(cout, generator=g), 0.05 * torch.randn(cout, generator=g), 0.1 * torch.randn(cout, generator=g),
          1 + 0.2 * torch.rand(cout, generator=g)]
    x = torch.randn((B, cin, H, W), generator=g)
    if "nobn" in opt:
        bn = None
    conv = Conv2d(w.numpy(), None if bn is None else [t.numpy() for t in bn], stride, pad)
    xd = x.to(cuda_dev)
    ref = F.conv2d(xd.double(), w.to(cuda_dev).double(), stride=stride, padding=pad)
    if bn is not None:
        ref = F.batch_norm(ref, bn[2].to(cuda_dev).double(), bn[3].to(cuda_dev).double(), bn[0].to(cuda_dev).double(),
                           bn[1].to(cuda_dev).double(), training=False, eps=1e-5)
    res = torch.randn(ref.shape, generator=g).to(cuda_dev)
    ref = ref + res.double()
    ref = (F.relu(ref) if relu else ref).float().permute(0, 2, 3, 1).contiguous()
    x_nhwc = xd.permute(0, 2, 3, 1).contiguous()
    res_nhwc = res.permute(0, 2, 3, 1).contiguous()
    y0 = conv(x_nhwc, res_nhwc, relu=relu, mode=0)
    scale = ref.abs().max().item()
    assert (y0 - ref).abs().max().item() / scale < 5e-6, "SIMT fp32"   # fp32 FMA accumulation over K up to 4608
    if cin % 32 == 0 and cout % 64 == 0 and k in (1, 3):
        y1 = conv(x_nhwc, res_nhwc, relu=relu, mode=1)
        err = (y1 - ref).abs().max().item() / scale
        assert err < 1e-5, "wgmma 3xTF32 rel err %g" % err   # tensor-core fp32 accumulation truncates; see conv_wgmma.cuh
        print("tc err", case, relu, err)


F16_CASES = [  # cin, cout, k, stride, pad, B, H, W, residual   (f16x3 kernel: Cin % 64 == 0, Cout % 64 == 0)
    (64, 64, 1, 1, 0, 2, 40, 48, False),       # N tile 64, one k-block per tile
    (64, 64, 3, 1, 1, 4, 128, 160, False),     # N tile 64, 9 k-blocks, 640 tiles: ring wrap-around
    (64, 256, 1, 1, 0, 4, 96, 128, True),      # N tile 128 + residual (K < 512)
    (256, 64, 1, 1, 0, 2, 37, 53, False),      # ragged tiles
    (128, 128, 3, 2, 1, 2, 64, 64, False),     # stride-2 3x3
    (128, 512, 1, 1, 0, 2, 33, 47, True),
    (256, 512, 1, 2, 0, 2, 33, 47, False),     # stride-2 projection, K = 256: N tile 128
    (512, 1024, 1, 2, 0, 2, 32, 32, False),    # K = 512, no residual
    (256, 256, 3, 1, 1, 3, 32, 32, False),     # K = 2304
    (512, 512, 3, 1, 1, 2, 20, 24, False),     # K = 4608: 72 k-blocks
    (512, 2048, 1, 1, 0, 2, 16, 16, True),     # residual, N tile 128
    (1024, 256, 1, 1, 0, 2, 33, 17, False),
    (2048, 512, 1, 1, 0, 5, 16, 16, False),    # K = 2048, 5 images
    (256, 128, 3, 1, 1, 2, 19, 27, False, "nobn"),   # no bias: the IRNet head / classifier epilogue
]


@pytest.mark.parametrize("case,relu", _with_relu(F16_CASES))
def test_conv_f16x3_vs_torch(cuda_dev, case, relu):
    """conv_wg_kernel<f16x3> (mode 2: fp16 hi/lo split operands, fp32 accumulation) against fp64 torch.  Same tolerance as the 3xTF32
    kernels: fp16 and tf32 carry the same 11 significant bits, the split keeps ~22 per operand."""
    from conftest import record
    cin, cout, k, stride, pad, B, H, W, with_res, *opt = case
    g = torch.Generator().manual_seed(cin * 11 + cout + k)
    w = torch.randn((cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5
    bn = [1 + 0.1 * torch.randn(cout, generator=g), 0.05 * torch.randn(cout, generator=g), 0.1 * torch.randn(cout, generator=g),
          1 + 0.2 * torch.rand(cout, generator=g)]
    if "nobn" in opt:
        bn = None
    x = torch.randn((B, cin, H, W), generator=g)
    conv = Conv2d(w.numpy(), None if bn is None else [t.numpy() for t in bn], stride, pad)
    xd = x.to(cuda_dev)
    ref = F.conv2d(xd.double(), w.to(cuda_dev).double(), stride=stride, padding=pad)
    if bn is not None:
        ref = F.batch_norm(ref, bn[2].to(cuda_dev).double(), bn[3].to(cuda_dev).double(), bn[0].to(cuda_dev).double(),
                           bn[1].to(cuda_dev).double(), training=False, eps=1e-5)
    res = torch.randn(ref.shape, generator=g).to(cuda_dev) if with_res else None
    if with_res:
        ref = ref + res.double()
    ref = (F.relu(ref) if relu else ref).float().permute(0, 2, 3, 1).contiguous()
    x_nhwc = xd.permute(0, 2, 3, 1).contiguous()
    y = conv(x_nhwc, None if res is None else res.permute(0, 2, 3, 1).contiguous(), relu=relu, mode=2)
    scale = ref.abs().max().item()
    err = (y - ref).abs().max().item() / scale
    bias = ((y - ref).double().sum() / ref.double().abs().sum()).item()       # accumulation truncation shows up as a systematic shrink
    record("conv_f16x3", case=list(case), relu=relu, rel_err=err, signed_bias=bias)
    assert err < 1e-5, "f16x3 rel err %g" % err
