"""CPU side of tests/test_backbone_stages_gpu.py: the workspace mirror against the library's workspace size, and the
stage rules against the float64 emulation of the split path (tests/backbone_ref.py) with and without defects.

The split rule must pass the clean emulation and fail each defect -- hi*lo or lo*hi product dropped, lo plane of the
output not stored, the remainder channels of a 196-channel input multiplied hi*hi only -- by at least 10x, judged
against the CPU fp32 oracle.  So the per-stage gate catches the bugs the end-to-end bound lets through, without a GPU.
The fp16 rule's accumulation term is shown to be needed: an exactly rounded fp32 accumulation of the fp16 operands
(what the fp16 kernels compute) lands more than one fp16 ulp from fp16(ref) at some outputs, yet passes the rule."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import backbone_ref as S
from loftr_b200 import _lib
from loftr_b200.loftr import TensorCoreBackbone

STAGES = {name: steps for name, _, steps in S.STAGES}
# stages reading a 196-channel activation: 3x3 halo (1/4 and 1/2 resolution), strided 1x1, FPN lateral with upsample
DEFECT_STAGES = ["l2.2", "l2.3", "l3.down", "l2_out", "l1_out2.0"]


@pytest.mark.parametrize("d2,d3", S.GRID_WIDTHS)
def test_workspace_mirror_matches_the_library(d2, d3):
    """carve_bb's layout as tests/backbone_ref.py mirrors it sums to the library's workspace size - 256"""
    m = S.make_backbone(d2, d3, "cpu")
    w, _ = TensorCoreBackbone(m, precision="fp16")._build()   # the workspace size reads only the layer widths
    lib = _lib.load()
    for n, h, wd in S.GRID_SHAPES:
        for planes, size in ((2, lib.lb_backbone_workspace_bytes), (1, lib.lb_backbone_workspace_bytes_fp16)):
            layout, total = S.workspace_layout(n, h, wd, (128, d2, d3), planes)
            assert total + 256 == size(C.byref(w), n, h, wd), (n, h, wd, planes)
            assert all((e[0] % 256, (e[1] or 0) % 256) == (0, 0) for e in layout.values())


@functools.lru_cache(maxsize=None)
def _emulated(precision):
    """The shipped widths on one 72 x 88 image: every buffer as the emulated kernels would store it"""
    m = S.make_backbone(196, 256, "cpu")
    rs = np.random.RandomState(5)
    bufs = {"image": torch.from_numpy(rs.uniform(0, 1, (1, 1, 72, 88))).double()}
    for name, _, steps in S.STAGES:
        if precision == "split":
            y = S.split_stage(m, steps, bufs.__getitem__)
        else:
            y = S.run_stage(m, steps, bufs.__getitem__, torch.float64, "fp16", store=S.r16)
            y = y if steps[-1][6] == "feat_f" else S.r16(y)
        bufs[steps[-1][6]] = y
    return m, bufs


@pytest.mark.parametrize("stage", DEFECT_STAGES)
def test_split_rule_catches_each_defect(stage):
    m, bufs = _emulated("split")
    steps = STAGES[stage]
    with torch.no_grad():
        ref = S.run_stage(m, steps, bufs.__getitem__, torch.float64)
        oracle = S.run_stage(m, steps, bufs.__getitem__, torch.float32)
        ok, clean = S.split_rule(S.split_stage(m, steps, bufs.__getitem__), ref, oracle)
        assert ok, (stage, clean)
        for defect in S.DEFECTS:
            got = S.split_stage(m, steps, bufs.__getitem__, defect)
            _, stats = S.split_rule(got, ref, oracle)
            assert stats["ratio"] >= 10, (stage, defect, stats)
            if stage in S.FINDING_STAGES:   # the bound of the listed H100 finding still catches it
                _, stats = S.split_rule(got, ref, oracle, S.FINDING_FACTOR)
                assert stats["ratio"] >= 2, (stage, defect, stats)


def test_fp16_rule_needs_its_accumulation_term():
    m, bufs = _emulated("fp16")
    worst_ulps = 0.0
    with torch.no_grad():
        for name, _, steps in S.STAGES:
            if steps[-1][6] == "feat_f":
                continue
            ref = S.run_stage(m, steps, bufs.__getitem__, torch.float64, "fp16", store=S.r16)
            oracle = S.run_stage(m, steps, bufs.__getitem__, torch.float32, "fp16", store=S.r16)
            ok, stats = S.fp16_rule(S.r16(oracle).double(), ref, oracle)
            assert ok, (name, stats)
            worst_ulps = max(worst_ulps, stats["max_ulps"])
            # an fp16 store that truncates instead of rounding to nearest differs at far more than 1 % of the values
            r16 = S.r16(ref)
            trunc = torch.where(r16.abs() > ref.abs(), r16 - torch.sign(r16) * S.fp16_ulp(r16), r16)
            assert not S.fp16_rule(trunc, ref, oracle)[0], name
    assert worst_ulps > 1
