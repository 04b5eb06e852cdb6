"""CPU-side checks of `LoFTR.match_points` (DESIGN.md §17): the numpy statement of its rounding rules on hand-computed
points, argument validation before any launch, the guard against a library without its two entries and their ABI
binding."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import loftr_b200
import util
from loftr_b200 import _lib
from points_ref import image1_centres, query_cells

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HW_I, HW_C, HW_F = (96, 128), (12, 16), (48, 64)   # s_c = 8, s_f = 2, stride = 4


@pytest.mark.parametrize("px, cx, fx", [
    (3.999, 0, 2),     # 3.999 / 8 + 0.5 < 1; 3.999 / 2 + 0.5 = 2.4995
    (4.0, 1, 2),       # exactly half a cell rounds up, not to even
    (4.001, 1, 2),
    (12.0, 2, 6),      # 1.5 cells -> 2 (banker's rounding would give 2 as well), 6 fine pixels
    (20.0, 3, 10),     # 2.5 cells -> 3 (banker's rounding: 2)
    (0.0, 0, 0),
    (127.0, 15, 63),   # W0 - 1: the last cell and fine pixel (16 and 64 before the clamp)
])
def test_cells_and_fine_centres_round_half_up(px, cx, fx):
    inside, cell, f0 = query_cells([[px, 40.0]], None, HW_I, HW_C, HW_F)
    assert inside.tolist() == [True]
    assert cell.tolist() == [[cx, 5]] and f0.tolist() == [[fx, 20]]


@pytest.mark.parametrize("px", [-0.5, 127.5, 128.0, float("nan"), float("inf"), -1e-3])
def test_points_outside_the_image_are_not_inside(px):
    inside, cell, f0 = query_cells([[px, 10.0], [10.0, px]], None, HW_I, HW_C, HW_F)
    assert inside.tolist() == [False, False]
    assert (cell == 0).all() and (f0 == 0).all()


def test_last_row_and_corner():
    inside, cell, f0 = query_cells([[127.0, 95.0], [0.0, 95.0], [126.9, 94.9]], None, HW_I, HW_C, HW_F)
    assert inside.all()
    assert cell.tolist() == [[15, 11], [0, 11], [15, 11]]
    assert f0.tolist() == [[63, 47], [0, 47], [63, 47]]


def test_valid0_mask0_and_scale0():
    mask0 = np.ones(HW_C, bool)
    mask0[5, 2] = False
    pts = [[16.0, 40.0], [24.0, 40.0], [24.0, 40.0]]
    inside, cell, _ = query_cells(pts, [True, True, False], HW_I, HW_C, HW_F, mask0=mask0)
    assert inside.tolist() == [False, True, False]      # masked cell, answered, valid0 false
    # source pixels: p / scale0 = (16, 40) -> cell (2, 5)
    inside, cell, f0 = query_cells([[32.0, 60.0]], None, HW_I, HW_C, HW_F, scale0=[2.0, 1.5])
    assert inside.tolist() == [True] and cell.tolist() == [[2, 5]] and f0.tolist() == [[8, 20]]


def test_image1_centres_keep_the_sub_cell_offset():
    # cell (3, 2), f0 = (13, 7): d = (1, -1); j = (5, 4) in a 16-wide image1 grid -> f1 = (21, 15)
    f1 = image1_centres([[3, 2]], [[13, 7]], [4 * 16 + 5], 16, 4)
    assert f1.tolist() == [[21, 15]]
    # a grid point has d = 0: f1 = stride * j
    inside, cell, f0 = query_cells([[8.0 * 5, 8.0 * 3]], None, HW_I, HW_C, HW_F)
    assert image1_centres(cell, f0, [7], 16, 4).tolist() == [[28, 0]]


# ------------------------------------------------------------------------------------------------ validation
def _model():
    return loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).eval()


def _data(n=2, **extra):
    return {"image0": torch.zeros(n, 1, 96, 128), "image1": torch.zeros(n, 1, 96, 128), **extra}


@pytest.mark.parametrize("points, err, msg", [
    (torch.zeros(2, 4, 2, dtype=torch.float64), TypeError, "float32"),
    (np.zeros((2, 4, 2), np.float32), TypeError, "float32"),
    (torch.zeros(2, 4), ValueError, r"\[N, Q, 2\]"),
    (torch.zeros(3, 4, 2), ValueError, r"\[N, Q, 2\] with N = 2"),
    (torch.zeros(2, 4, 3), ValueError, r"\[N, Q, 2\]"),
])
def test_points_are_validated_before_any_launch(points, err, msg):
    model = _model()
    with pytest.raises(err, match=msg):
        model.match_points(_data(), points)


def test_valid0_scales_masks_and_devices_are_validated():
    model = _model()
    pts = torch.zeros(2, 4, 2)
    with pytest.raises(TypeError, match="valid0 must be a bool"):
        model.match_points(_data(), pts, torch.ones(2, 4, dtype=torch.uint8))
    with pytest.raises(ValueError, match=r"valid0 must be \[N, Q\] = \(2, 4\)"):
        model.match_points(_data(), pts, torch.ones(2, 5, dtype=torch.bool))
    with pytest.raises(ValueError, match="scale0 and scale1 together"):
        model.match_points(_data(scale0=torch.ones(2, 2)), pts)
    with pytest.raises(ValueError, match="mask0 and mask1 together"):
        model.match_points(_data(mask1=torch.ones(2, 12, 16, dtype=torch.bool)), pts)
    with pytest.raises(ValueError, match="must hold `image1`"):
        model.match_points({"image0": torch.zeros(2, 1, 96, 128)}, pts)
    # well-formed arguments on the host: the device check is what stops them (Q = 0 included)
    for q in (4, 0):
        with pytest.raises(ValueError, match="`image0` must be a CUDA tensor"):
            model.match_points(_data(), torch.zeros(2, q, 2), torch.ones(2, q, dtype=torch.bool))


@pytest.mark.parametrize("version", [110, 109])
def test_match_points_refuses_a_library_without_its_entries(monkeypatch, version):
    util.old_library(monkeypatch, version)   # a build from before the point entries: no lb_coarse_query / centre gather
    assert _lib.POINTS_ENTRIES == ("lb_coarse_query", "lb_fine_preprocess_centres")
    model = _model()
    with pytest.raises(RuntimeError, match=rf"match_points needs lb_coarse_query, which .* \(version {version}\) does "
                                           "not export"):
        model.match_points({}, torch.zeros(1, 1, 2))
    cm = model.coarse_matching
    with pytest.raises(RuntimeError, match="match_points needs lb_coarse_query"):
        cm.query(None, None, 256, 1, 4, 4, 256, {}, None, None, torch.zeros(1, 1, 2))
    # every other path still accepts such a library: the forward's coarse stage is not what it stops
    with pytest.raises(AttributeError):
        cm.run(None, None, 256, 1, 4, 4, 256, {})


def test_load_binds_the_point_entries_only_where_exported(monkeypatch, tmp_path):
    # the shipped build exports both and reports the version of its newest versioned entry
    lib = _lib.load()
    assert lib.lb_version() == _lib.GEMM_FP16_VERSION
    for name in _lib.POINTS_ENTRIES:
        assert name not in _lib._SINCE
        assert _lib.SIGNATURES[name][1] == getattr(lib, name).argtypes
    _lib.require_entries(_lib.POINTS_ENTRIES, "match_points")
    old = util.load_without(monkeypatch, _lib.POINTS_ENTRIES)
    assert not any(hasattr(old, n) for n in _lib.POINTS_ENTRIES)
    assert old.lb_coarse_match.argtypes == _lib.SIGNATURES["lb_coarse_match"][1]
    with pytest.raises(RuntimeError, match=r"needs lb_coarse_query.*\(version 110\)"):
        _lib.require_entries(_lib.POINTS_ENTRIES, "match_points")


def test_point_entries_check_their_arguments():
    lib = _lib.load()
    names = {lib.lb_timing_tag_name(i).decode() for i in range(lib.lb_timing_num_tags())}
    assert "match_query" in names
    a, q = _lib.LbCoarseMatchArgs(), _lib.LbCoarseQueryArgs()
    assert lib.lb_coarse_query(C.byref(a), C.byref(q), 3, None, 0, None) != 0
    assert b"operand_planes must be 1 (fp16) or 2 (split)" in lib.lb_last_error()
    assert lib.lb_coarse_query(C.byref(a), C.byref(q), 2, None, 0, None) == 0   # Q = 0: nothing to do
    f = _lib.LbFinePreprocessArgs()
    f.M = 4
    assert lib.lb_fine_preprocess_centres(C.byref(f), None, None, None, 0, None) != 0
    assert b"centres and inside are required" in lib.lb_last_error()


def test_query_struct_layout_matches_header():
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "loftr_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct LbCoarseQueryArgs \{(.*?)\} LbCoarseQueryArgs;", header, re.S).group(1)
    names = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        first, *rest = decl.split(",")
        names += [re.findall(r"[A-Za-z_0-9]+", first)[-1]] + [re.findall(r"[A-Za-z_0-9]+", r)[-1] for r in rest]
    assert names == [f[0] for f in _lib.LbCoarseQueryArgs._fields_]
