"""Every stage of the tensor-core backbone against float64, from the kernels' own stored inputs.

One forward of lb_backbone_forward (split) or lb_backbone_forward_fp16 runs into a workspace the test allocates; the
mirror of `carve_bb` in tests/backbone_ref.py then reads every activation back, and each stage (one convolution,
or two where the first one's output is overwritten later: t1, t2, t3) is recomputed from the inputs the kernels stored,
residual and upsample addends included.  So a stage's error is its own, and a failure names its layer and kernel
class: the stem (conv_stem7x7_tc), the halo convolution (conv3x3_halo_kernel: every stride-1 3x3), the implicit GEMM
(gemm_split_kernel: the strided 3x3 and the 1x1 convolutions) and the FPN upsample-add epilogue of the two lateral 1x1
convolutions.

Rules (DESIGN.md §2, §15):
- split path: ref is the stage in float64 with the fp32 weights, oracle the same stage in fp32 (TF32 off).
  max|kernel - ref| <= 4 max|oracle - ref| + 2^-22 max|ref|: the dense-output rule of test_kernel_edges_gpu.py plus
  the rounding of the stored hi + lo output.
- fp16 path, stored planes: ref uses the weights fp16(w * 2^e) * 2^-e and the stored fp16 inputs, rounded to fp16
  only where the kernel stores.  Every stored value is within one fp16 ulp of fp16(ref) plus 4 max|oracle - ref|
  (oracle: the same fp16 operands in fp32), and at most 1 % of the values differ from fp16(ref) at all.  The second
  term is the fp32 accumulation: where the output is much smaller than the products it sums (near zero, and behind a
  chain's fp16 intermediate, whose one-ulp flips the second convolution amplifies) an exactly rounded fp32
  accumulation already lands several ulps from fp16(ref); tests/test_backbone_stages_cpu.py shows that with an fp32
  emulation of the kernel.
- fp16 path, the fp32 maps feat_c and feat_f: the split rule, with the fp16 operands as the exact operands.
- fp16 path, a chain of two convolutions: the split rule with 2^-11 (one fp16 rounding) as the storage term.
The 3x3 stages are a listed finding (FINDING_STAGES in tests/backbone_ref.py): 16x the oracle's error instead of 4x.

The grid covers a 1 x 1 map at 1/8 (upsampled from one pixel), partial 8 x 16 tiles at every level with three images
(a halo leaking across images shows at their borders), one-row and one-column images, multi-tile CTA sequences and the
benchmark size, at the shipped widths and at three of test_backbone_widths_gpu.WIDTHS (channel remainders,
zero-padded last channel blocks, Cout on both sides of 128 and 200).  Every stage's ratio to its bound is recorded."""
import pytest
import torch

import backbone_ref as S
import util

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

SHAPES = S.GRID_SHAPES
# (d2, d3): the shipped ResNetFPN_8_2 widths (d1 = 128 always) and three of test_backbone_widths_gpu.WIDTHS
WIDTHS = S.GRID_WIDTHS


@pytest.mark.parametrize("precision", ["split", "fp16"])
@pytest.mark.parametrize("d2,d3", WIDTHS)
@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_backbone_stages_match_fp64(shape, d2, d3, precision):
    from loftr_b200.loftr import TensorCoreBackbone
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    n, h, w = shape
    m = S.make_backbone(d2, d3, DEV)
    img = S.image(shape, d2 + d3 + h + w)
    fp16 = precision == "fp16"
    ws, feat_c, feat_f = S.backbone_forward(TensorCoreBackbone(m, precision=precision), img)
    layout, total = S.workspace_layout(n, h, w, (128, d2, d3), 1 if fp16 else 2)
    assert total + 256 == ws.numel(), "tests/backbone_ref.py no longer mirrors carve_bb"
    stored = {"image": img.double(), "feat_c": feat_c.permute(0, 3, 1, 2).double(),
              "feat_f": feat_f.permute(0, 3, 1, 2).double()}

    def get(name):
        if name not in stored:
            stored[name] = S.decode(ws, layout[name])
        return stored[name]

    weights = "fp16" if fp16 else "fp32"
    failed = []
    tag = "backbone_stage_%s_%dx%d_%dx%dx%d" % (precision, d2, d3, n, h, w)
    with torch.no_grad():
        for name, cls, steps in S.STAGES:
            ref = S.run_stage(m, steps, get, torch.float64, weights, store=S.r16 if fp16 else None)
            oracle = S.run_stage(m, steps, get, torch.float32, weights, store=S.r16 if fp16 else None)
            out = steps[-1][6]
            checks = [(out, get(out))] if out != "feat_f" else []
            if out in S.FP32_OUTPUTS:
                checks.append((S.FP32_OUTPUTS[out], get(S.FP32_OUTPUTS[out])))
            finding = name in S.FINDING_STAGES
            factor = S.FINDING_FACTOR if finding else S.FACTOR
            for buf, got in checks:
                assert got.shape == ref.shape, (name, buf, got.shape, ref.shape)
                if not fp16 or buf.startswith("feat"):
                    rule, ok, stats = "split", *S.split_rule(got, ref, oracle, factor)
                    strict = S.split_rule(got, ref, oracle)[1]["ratio"]
                elif len(steps) == 2:
                    # a chain's fp16 intermediate: the kernel's own one-ulp differences there are amplified by the
                    # second convolution, so its output is judged like a map with one fp16 storage rounding
                    rule, ok, stats = "fp16_chain", *S.split_rule(got, ref, oracle, factor, S.FP16_STORE_TERM)
                    strict = S.split_rule(got, ref, oracle, S.FACTOR, S.FP16_STORE_TERM)[1]["ratio"]
                else:
                    rule, ok, stats = "fp16", *S.fp16_rule(got, ref, oracle, factor,
                                                          S.FINDING_SHARE if finding else S.FP16_DIFF_SHARE)
                    strict = S.fp16_rule(got, ref, oracle)[1]["ratio"]
                util.record(f"{tag}_{name}_{buf}", {"class": cls, "rule": rule, "finding": finding,
                                                    "ratio_at_4x": strict, **stats})
                if not ok:
                    failed.append(f"{name} -> {buf} ({cls}, {rule} rule): " +
                                  ", ".join(f"{k} {v:.3e}" for k, v in stats.items()))
    assert not failed, "; ".join(failed)
