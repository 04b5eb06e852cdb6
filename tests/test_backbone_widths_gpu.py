"""The backbone convolutions at layer2 / layer3 widths other than the shipped [128, 196, 256]: `ResNetFPN(128, [128, d2,
d3])` with random BatchNorm statistics through TensorCoreBackbone, both precisions, against the float64 module.

`TensorCoreBackbone.supported()` accepts any d2 up to 256 and any d3 up to 256 that is divisible by 4, and
`backbone_impl="auto"` then picks the tensor-core backbone, so every such width has to run.  The pairs below give the halo convolution Cin 40, 64,
72, 80, 81, 136, 160, 193, 208, 209 and 256: 1, 2, 3 and 4 halos per tile, tap-major and channel-block-major order,
channel remainders r = 1, 8 and 16 and zero-padded last blocks (Cin 40, 81, 160, 209), and output tiles of 128, 200 and
256 columns with Cout on both sides of 128, 200 and 208 (208 is the widest gemm_split_kernel tile below 256).
tests/test_pipeline_coverage_cpu.py checks that these categories stay covered.

Bounds: the split path is held to 1e-4 of each output map's scale (test_backbone_halo_convs_match_fp64), the fp16 path
to twice the error of its float64 emulation plus 1e-6 of the scale (test_fp16_backbone_error_is_that_of_its_semantics)."""
import copy

import pytest
import torch

import backbone_ref as B
import loftr_b200
import util

DEV = "cuda:0"
gpu = pytest.mark.gpu

# (d2, d3)
WIDTHS = [(72, 256), (80, 136), (81, 208), (136, 200), (160, 72), (193, 80), (209, 64), (40, 160), (208, 40),
          (256, 256)]
# at 8 x 136 x 200 the 1/2- and 1/4-resolution layers run several tiles per CTA
BATCH8 = [(81, 208), (136, 200), (193, 80), (209, 64)]
SHAPES = [(1, 16, 16), (2, 88, 72)]
# activation rows padded to a multiple of 8 channels: 81 -> 88, 193 -> 200, 209 -> 216
PADDED = [(81, 208), (193, 80), (209, 64)]


@gpu
@pytest.mark.parametrize("d2,d3,shape", [(*d, s) for d in WIDTHS for s in SHAPES] + [(*d, (8, 136, 200)) for d in BATCH8])
def test_backbone_widths_match_fp64(d2, d3, shape):
    from loftr_b200.loftr import TensorCoreBackbone
    m = B.make_backbone(d2, d3, DEV)
    assert TensorCoreBackbone.supported(m)
    img = B.image(shape, d2 + d3)
    with torch.no_grad():
        ex = copy.deepcopy(m).double()(img.double())
        emu = B.forward_f64(m, img)
    split = B.backbone_forward(TensorCoreBackbone(m), img)[1:]
    fp16 = B.backbone_forward(TensorCoreBackbone(m, precision="fp16"), img)[1:]
    stats, failed = {}, []
    for name, g_split, g_fp16, x, e in zip(("coarse", "fine"), split, fp16, ex, emu):
        scale = x.abs().max().item()
        err = (g_split.permute(0, 3, 1, 2).double() - x).abs().max().item()
        err16 = (g_fp16.permute(0, 3, 1, 2).double() - x).abs().max().item()
        err_emu = (e - x).abs().max().item()
        stats.update({f"{name}_scale": scale, f"{name}_split_err_over_bound": err / (1e-4 * scale),
                      f"{name}_fp16_err_over_bound": err16 / (2 * err_emu + 1e-6 * scale)})
        if not err <= 1e-4 * scale:
            failed.append(f"split {name}: {err:.3e} (scale {scale:.3e})")
        if not err16 <= 2 * err_emu + 1e-6 * scale:
            failed.append(f"fp16 {name}: {err16:.3e} vs emulation {err_emu:.3e} (scale {scale:.3e})")
    util.record("backbone_widths_%dx%d_%dx%dx%d" % (d2, d3, *shape), stats)
    assert not failed, "; ".join(failed)


@gpu
@pytest.mark.parametrize("precision", ["split", "fp16"])
@pytest.mark.parametrize("d2,d3", PADDED)
def test_backbone_widths_ignore_padding_and_batch_position(d2, d3, precision):
    """The channels between a layer's width and its padded row stride are never written: a NaN-filled workspace gives
    the bits of a zeroed one.  An image alone gives the bits it gets inside a batch."""
    from loftr_b200.loftr import TensorCoreBackbone
    tc = TensorCoreBackbone(B.make_backbone(d2, d3, DEV), precision=precision)
    batch = B.image((3, 88, 72), 7)
    _, zc, zf = B.backbone_forward(tc, batch, 0)
    _, nc, nf = B.backbone_forward(tc, batch, 0xFF)
    assert torch.isfinite(zc).all() and torch.isfinite(zf).all()
    assert torch.equal(zc, nc) and torch.equal(zf, nf)
    for i in (0, 2):
        _, c, f = B.backbone_forward(tc, batch[i:i + 1].contiguous(), 0xFF)
        assert torch.equal(c[0], zc[i]) and torch.equal(f[0], zf[i]), i


@gpu
@pytest.mark.parametrize("d3", [130, 201])
def test_coarse_width_not_divisible_by_4_cannot_run(d3):
    """feat_c is stored as fp32 NHWC rows of d3 values through a TMA map, whose row stride must be a multiple of 16
    bytes: d3 % 4 != 0 fails there, which is why `supported()` refuses such widths."""
    from loftr_b200.loftr import TensorCoreBackbone
    m = B.make_backbone(196, d3, DEV)
    assert not TensorCoreBackbone.supported(m)
    with pytest.raises(RuntimeError, match="not a multiple of 16"):
        B.backbone_forward(TensorCoreBackbone(m), B.image((1, 16, 16), 3))


@pytest.mark.parametrize("d3", [130, 201])
def test_auto_keeps_the_torch_backbone_for_a_coarse_width_not_divisible_by_4(d3):
    cfg = loftr_b200.get_cfg("indoor_ds")
    cfg["resnetfpn"]["block_dims"] = [128, 196, d3]
    assert loftr_b200.LoFTR(cfg).backbone_impl == "torch"
    for impl in ("b200", "b200_fp16"):
        with pytest.raises(ValueError, match="tensor-core backbone"):
            loftr_b200.LoFTR(cfg, backbone_impl=impl)
