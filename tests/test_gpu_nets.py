"""CAM / EdgeDisplacement forward on the GPU against the reference's outputs (golden fixtures made
by the unmodified reference on CPU, IEEE fp32).  Tolerance: 1e-4 max-abs on the max-normalised CAM
(BASELINE.json north_star), stated per assertion."""
import numpy as np
import pytest
import torch

from conftest import golden_path, record
from irn_b200 import synth
from irn_b200.cam import CAM
from irn_b200.irn import EdgeDisplacement

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cam_model(cuda_dev):
    m = CAM()
    m.load_state_dict(synth.cam_state_dict(), strict=True)
    m.eval()
    return m


@pytest.fixture(scope="module")
def irn_model(cuda_dev):
    m = EdgeDisplacement()
    m.load_state_dict(synth.irn_state_dict(), strict=False)
    m.eval()
    return m


@pytest.mark.parametrize("mode", [1, 2], ids=["tf32x3", "f16x3"])
def test_cam_forward_vs_reference(cuda_dev, cam_model, mode):
    g = np.load(golden_path("cam_forward.npz"))
    cam_model.set_conv_mode(mode)
    for i in range(3):
        y = cam_model(torch.from_numpy(g["x%d" % i]).to(cuda_dev)).cpu().numpy()
        ref = g["y%d" % i]
        assert y.shape == ref.shape
        scale = ref.max()
        err = np.abs(y - ref).max() / scale
        record("cam_forward_vs_reference", input=list(g["x%d" % i].shape[-2:]), normalised_err=err, conv_mode=mode)
        assert err < 1e-4, "normalised CAM err %g" % err
    cam_model.set_conv_mode(None)


def test_cam_batch_equals_single(cuda_dev, cam_model):
    g = np.load(golden_path("cam_forward.npz"))
    x = torch.from_numpy(g["x0"]).to(cuda_dev)
    xb = torch.cat([x, x.flip(0), x], 0)          # three pairs
    yb = cam_model.forward_batch(xb)
    y = cam_model(x)
    assert torch.equal(yb[0], y) and torch.equal(yb[2], y)
    # flipping the pair flips the CAM (SURVEY.md section 4 property)
    assert torch.allclose(yb[1], y.flip(-1), atol=1e-5)


def test_edge_displacement_vs_reference(cuda_dev, irn_model):
    g = np.load(golden_path("irn_forward.npz"))
    for i in range(3):
        if ("x%d" % i) in g:
            x = g["x%d" % i]
        else:
            x = synth.normalize_image(synth.image(200 + i, 512, 512))
            x = np.stack([x, x[..., ::-1].copy()])
        e, d = irn_model(torch.from_numpy(x).to(cuda_dev))
        assert e.shape == g["edge%d" % i].shape and d.shape == g["dp%d" % i].shape
        e_err = np.abs(e.cpu().numpy() - g["edge%d" % i]).max()
        d_err = np.abs(d.cpu().numpy() - g["dp%d" % i]).max()
        d_max = np.abs(g["dp%d" % i]).max()
        record("edge_displacement_vs_reference", input=list(x.shape[-2:]), edge_err=e_err, dp_err=d_err, dp_absmax=d_max)
        assert e_err < 1e-4                               # edge is a sigmoid output in (0,1): absolute = relative to full scale
        assert d_err < 1e-4, "dp err %g (|dp|max %g)" % (d_err, d_max)       # absolute, in stride-4 pixels 


def test_state_dict_keys_match_reference_format(cam_model, irn_model):
    assert len(cam_model.state_dict()) == 956 and len(irn_model.state_dict()) == 1035   # SURVEY.md D10
