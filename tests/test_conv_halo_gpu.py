"""The stride-1 3x3 backbone convolutions (conv3x3_halo_kernel: the input halo loaded once per channel block) through
lb_backbone_forward: every layer class of the network -- Cin 128 / 196 / 256 with the 196 = 3 * 64 + 4 channel
remainder, Cout tiles 128 / 208 / 256, BatchNorm, residual and FPN paths -- against the float64 PyTorch module, at
batch 1 and 16 and at sizes whose 1/2, 1/4 and 1/8 grids are not multiples of the 8 x 16 output tile (a 16 x 16
image leaves 2 x 2 pixels at 1/8: the halo is mostly zero fill)."""
import copy

import pytest
import torch

import backbone_ref as B
import util
from cases import CASES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("shape", [(1, 16, 16), (16, 136, 200), (1, 88, 72)])
def test_backbone_halo_convs_match_fp64(shape):
    from loftr_b200.loftr import TensorCoreBackbone
    n, h, w = shape
    model, _, _ = util.build_model(dict(CASES[0]), DEV)
    img = B.image(shape, 11)
    with torch.no_grad():
        ex_c, ex_f = copy.deepcopy(model.backbone).double()(img.double())
    tc = TensorCoreBackbone(model.backbone)
    _, got_c, got_f = B.backbone_forward(tc, img)
    for got, ex, name in ((got_c, ex_c, "coarse"), (got_f, ex_f, "fine")):
        scale = ex.abs().max().item()
        err = (got.permute(0, 3, 1, 2).double() - ex).abs().max().item()
        util.record(f"backbone_halo_{name}_{n}x{h}x{w}", {"err_over_scale": err / scale, "scale": scale})
        assert err <= 1e-4 * scale, f"{name}: {err:.3e} (scale {scale:.3e})"


def test_backbone_ignores_channel_padding():
    """Activation planes of 196 channels have a row stride of 200 elements; channels 196..199 are never written.  A
    workspace full of NaN must give the same bits as a zeroed one: the padding never reaches an MMA."""
    from loftr_b200.loftr import TensorCoreBackbone
    model, _, _ = util.build_model(dict(CASES[0]), DEV)
    img = B.image((2, 96, 136), 12)
    tc = TensorCoreBackbone(model.backbone)
    _, zc, zf = B.backbone_forward(tc, img, 0)
    _, nc, nf = B.backbone_forward(tc, img, 0xFF)
    assert torch.isfinite(nc).all() and torch.isfinite(nf).all()
    assert torch.equal(zc, nc) and torch.equal(zf, nf)
