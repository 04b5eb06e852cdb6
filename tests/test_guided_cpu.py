"""CPU-side checks of guided coarse matching (DESIGN.md §18): the shared guide validator and the callers that refuse a
guide, the binding of lb_coarse_match_guided by name and its argument errors, and self-checks of the
float64 guided reference (tests/guided_ref.py's admissibility under ref64.conf_matrix) against unguided ref64."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import guided_ref as G
import loftr_b200
import ref64 as R
import util
from loftr_b200 import _lib
from loftr_b200.loftr import CapturedMatcher, CoarseMatching, check_guide
from cases import build_cfg, build_cm_inputs


def _guide(n=2, **kw):
    g = {"kind": "fundamental", "model": torch.zeros(n, 3, 3), "radius": 8.0}
    g.update(kw)
    return g


@pytest.mark.parametrize("guide, exc, match", [
    ([1, 2], TypeError, "guide must be a dict"),
    ({"kind": "fundamental", "model": torch.zeros(2, 3, 3)}, ValueError, "exactly the keys"),
    (dict(_guide(), extra=1), ValueError, "exactly the keys"),
    (_guide(kind="affine"), ValueError, r"guide\['kind'\]"),
    (_guide(kind=1), ValueError, r"guide\['kind'\]"),
    (_guide(model=np.zeros((2, 3, 3), np.float32)), TypeError, r"guide\['model'\] must be a float32 tensor"),
    (_guide(model=torch.zeros(2, 3, 3, dtype=torch.float64)), TypeError, r"guide\['model'\] must be a float32"),
    (_guide(model=torch.zeros(3, 3, 3)), ValueError, r"guide\['model'\] must be \[N, 3, 3\] with N = 2"),
    (_guide(model=torch.zeros(2, 9)), ValueError, r"guide\['model'\] must be \[N, 3, 3\]"),
    (_guide(model=torch.zeros(2, 3, 3, device="meta")), ValueError, r"guide\['model'\] is on meta"),
    (_guide(radius="8"), TypeError, r"guide\['radius'\] must be a real number"),
    (_guide(radius=True), TypeError, r"guide\['radius'\] must be a real number"),
    (_guide(radius=torch.tensor(8.0)), TypeError, r"guide\['radius'\] must be a real number"),
    (_guide(radius=0.0), ValueError, r"guide\['radius'\] must be finite and positive"),
    (_guide(radius=-1.0), ValueError, r"guide\['radius'\] must be finite and positive"),
    (_guide(radius=math.inf), ValueError, r"guide\['radius'\] must be finite and positive"),
    (_guide(radius=math.nan), ValueError, r"guide\['radius'\] must be finite and positive"),
], ids=["not_dict", "missing_key", "extra_key", "kind", "kind_int", "model_numpy", "model_f64", "model_n",
        "model_shape", "model_device", "radius_str", "radius_bool", "radius_tensor", "radius_0", "radius_neg",
        "radius_inf", "radius_nan"])
def test_validator_rejects(guide, exc, match):
    with pytest.raises(exc, match="match_features: .*" + match):
        check_guide(guide, 2, "cpu", 0.0, "match_features")


def test_validator_accepts_and_requires_thr_at_least_zero():
    model = torch.full((2, 3, 3), float("nan"))   # NaN entries are data, not an error: the pair is unguided
    for kind, code in (("fundamental", _lib.GUIDE_FUNDAMENTAL), ("homography", _lib.GUIDE_HOMOGRAPHY)):
        k, m, r = check_guide(_guide(kind=kind, model=model, radius=3), 2, torch.device("cpu"), 0.0, "forward")
        assert (k, r) == (code, 3.0) and m.is_contiguous() and m.data_ptr() == model.data_ptr()
    with pytest.raises(ValueError, match=r"forward: a guide needs match_coarse.thr >= 0 \(got -0.5\)"):
        check_guide(_guide(), 2, "cpu", -0.5, "forward")


def test_coarse_matching_reads_the_guide_through_its_arguments():
    """CoarseMatching.run validates data["guide"] (here: thr < 0) before it launches anything."""
    mc = build_cfg({"thr": -1.0, "match_type": "dual_softmax", "prefilter": False, "border_rm": 0})["match_coarse"]
    cm = CoarseMatching(mc).eval()
    hi = torch.zeros(8, 256, dtype=torch.float16)
    data = {"hw0_i": (16, 16), "hw0_c": (2, 2), "hw1_c": (2, 2), "guide": _guide(n=1)}
    with pytest.raises(ValueError, match="CoarseMatching: a guide needs match_coarse.thr >= 0"):
        cm.run(hi, hi, 256, 1, 4, 4, 256, data)


def test_match_points_and_captured_matcher_refuse_a_guide():
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).eval()
    with pytest.raises(ValueError, match=r"match_points: data\['guide'\] is not supported"):
        model.match_points({"image0": torch.zeros(1, 1, 8, 8), "image1": torch.zeros(1, 1, 8, 8), "guide": _guide(1)},
                           torch.zeros(1, 1, 2))
    cap = CapturedMatcher.__new__(CapturedMatcher)   # the guide is refused before the graph or the weights are read
    cap.graph = None
    with pytest.raises(ValueError, match=r"CapturedMatcher: data\['guide'\] is not supported"):
        cap({"image0": torch.zeros(1, 1, 8, 8), "guide": _guide(1)})


def test_guided_entry_is_bound_only_where_exported(monkeypatch):
    """lb_coarse_match_guided comes without a version step, found by name like the point entries (DESIGN.md §17):
    the shipped build exports and binds it; a build without it still loads, and only a guide is refused."""
    lib = _lib.load()
    assert _lib.GUIDE_ENTRIES == ("lb_coarse_match_guided",) and "lb_coarse_match_guided" not in _lib._SINCE
    assert lib.lb_coarse_match_guided.argtypes == _lib.SIGNATURES["lb_coarse_match_guided"][1]
    _lib.require_entries(_lib.GUIDE_ENTRIES, "guided matching")
    old = util.load_without(monkeypatch, _lib.GUIDE_ENTRIES)
    assert not hasattr(old, "lb_coarse_match_guided")
    assert old.lb_coarse_match_fp16.argtypes == _lib.SIGNATURES["lb_coarse_match_fp16"][1]   # the rest still binds
    with pytest.raises(RuntimeError, match=r"forward: guided matching needs lb_coarse_match_guided.*\(version 110\)"):
        check_guide(_guide(), 2, "cpu", 0.0, "forward")


def test_guided_entry_checks_its_arguments():
    lib = _lib.load()
    a = _lib.LbCoarseMatchArgs()
    model = torch.zeros(1, 9)
    cases = [(None, b"the guide model is null"),
             (_lib.LbCoarseGuide(_lib.GUIDE_FUNDAMENTAL, None, 8.0), b"the guide model is null"),
             (_lib.LbCoarseGuide(7, model.data_ptr(), 8.0), b"unknown guide kind 7")]
    cases += [(_lib.LbCoarseGuide(_lib.GUIDE_HOMOGRAPHY, model.data_ptr(), r), b"radius must be finite and positive")
              for r in (0.0, -2.0, math.inf, math.nan)]
    for g, msg in cases:
        assert lib.lb_coarse_match_guided(C.byref(a), None if g is None else C.byref(g), 0, 0, None, 0, None) != 0
        assert msg in lib.lb_last_error(), (g, lib.lb_last_error())
    g = _lib.LbCoarseGuide(_lib.GUIDE_FUNDAMENTAL, model.data_ptr(), 8.0)
    assert lib.lb_coarse_match_guided(C.byref(a), C.byref(g), -1, 0, None, 0, None) != 0
    assert b"max_per_pair must be 0" in lib.lb_last_error()
    assert lib.lb_coarse_match_guided(C.byref(a), C.byref(g), 0, 2, None, 0, None) != 0
    assert b"fp16 must be 0 (split) or 1" in lib.lb_last_error()


# ------------------------------------------------------------------------------------------------ oracle self-checks
def _cm_case(match_type, n=2, hw0c=(6, 7), hw1c=(5, 8), prefilter=True, masked=False):
    case = {"n": n, "hw0c": hw0c, "hw1c": hw1c, "amp": 3.0 if match_type == "sinkhorn" else 1.6, "frac": 0.6,
            "iseed": 5}
    if masked:
        case.update(valid0c=[(6, 5), (4, 7)], valid1c=[(5, 8), (5, 6)])
    inp = build_cm_inputs(case)
    mc = build_cfg({"thr": 0.0, "match_type": match_type, "prefilter": prefilter, "border_rm": 1})["match_coarse"]
    mc["skh_iters"], mc["dsmax_temperature"] = 3, 0.1
    return case, inp, mc


def _guided(inp, case, mc, adm, masked):
    (h0, w0), (h1, w1) = case["hw0c"], case["hw1c"]
    m0 = m1 = mk0 = mk1 = None
    if masked:
        mk0, mk1 = torch.as_tensor(inp["mask0"]), torch.as_tensor(inp["mask1"])
        m0, m1 = mk0.flatten(-2), mk1.flatten(-2)
    f0, f1 = R.f64(inp["feat_c0"]), R.f64(inp["feat_c1"])
    conf = R.conf_matrix(f0, f1, mc, m0, m1, 1.0, adm=None if adm is None else torch.as_tensor(adm))
    return conf, R.coarse_match(conf, mc, (h0 * 8, w0 * 8), (h0, w0), (h1, w1), mk0, mk1)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
def test_oracle_all_admissible_guide_equals_ref64(match_type, masked):
    case, inp, mc = _cm_case(match_type, masked=masked)
    n, (h0, w0), (h1, w1) = case["n"], case["hw0c"], case["hw1c"]
    p0, p1 = G.coarse_points(n, (h0, w0), 8.0), G.coarse_points(n, (h1, w1), 8.0)
    rs = np.random.RandomState(3)
    _, ref = _guided(inp, case, mc, None, masked)
    assert len(ref["b_ids"]) > 0
    for kind, model, radius in (("fundamental", rs.standard_normal((n, 3, 3)), 1e9),
                                ("homography", np.eye(3)[None].repeat(n, 0), 1e9),
                                ("homography", np.full((n, 3, 3), np.nan), 1.0)):
        adm, _ = G.admissible(kind, model, radius, p0, p1)
        assert adm.all()
        conf, got = _guided(inp, case, mc, adm, masked)
        for k in ref:
            assert torch.equal(got[k], ref[k]), (kind, k)


@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
def test_oracle_selects_admissible_pairs_only(match_type):
    case, inp, mc = _cm_case(match_type, hw0c=(9, 10), hw1c=(8, 11))
    n, (h0, w0), (h1, w1) = case["n"], case["hw0c"], case["hw1c"]
    scale0, scale1 = np.array([[1.5, 1.25], [1.0, 2.0]], np.float32), np.array([[0.75, 1.0], [2.0, 1.5]], np.float32)
    p0, p1 = G.coarse_points(n, (h0, w0), 8.0, scale0), G.coarse_points(n, (h1, w1), 8.0, scale1)
    H = np.array([[[1.0, 0.05, 3.0], [-0.02, 0.9, -4.0], [1e-4, 0.0, 1.0]]] * n, np.float32)
    F = np.array([[[0.0, -1e-3, 0.05], [1e-3, 0.0, -0.1], [-0.04, 0.1, 0.5]]] * n, np.float32)
    for kind, model, radius in (("homography", H, 20.0), ("fundamental", F, 6.0)):
        adm, margin = G.admissible(kind, model, radius, p0, p1)
        assert 0.05 < adm.mean() < 0.8, (kind, adm.mean())   # the band cuts through every pair's grid
        conf, got = _guided(inp, case, mc, adm, False)
        b, i, j = (got[k].numpy() for k in ("b_ids", "i_ids", "j_ids"))
        assert len(b) > 0 and adm[b, i, j].all()
        assert (conf.numpy()[~adm] == 0).all()
    # the float32 predicate in the expression the kernels evaluate, by hand for one cell pair of each kind
    x0, y0 = p0[0, 13]
    x1, y1 = p1[0, 30]
    l = [(F[0, k, 0] * x0 + F[0, k, 1] * y0) + F[0, k, 2] for k in range(3)]
    e = (l[0] * x1 + l[1] * y1) + l[2]
    assert G.admissible("fundamental", F, 6.0, p0, p1)[0][0, 13, 30] == (abs(e) <= np.float32(6.0) * np.sqrt(
        l[0] * l[0] + l[1] * l[1]))
    q = [(H[0, k, 0] * x0 + H[0, k, 1] * y0) + H[0, k, 2] for k in range(3)]
    dx, dy = q[0] / q[2] - x1, q[1] / q[2] - y1
    assert G.admissible("homography", H, 20.0, p0, p1)[0][0, 13, 30] == (dx * dx + dy * dy <= np.float32(400.0))


def test_oracle_line_through_nothing_and_homography_to_infinity_admit_nothing():
    p0, p1 = G.coarse_points(1, (3, 4), 8.0), G.coarse_points(1, (3, 4), 8.0)
    F = np.zeros((1, 3, 3), np.float32)
    F[0, 2, 2] = 1.0                  # l = (0, 0, 1) for every p0
    H = np.eye(3, dtype=np.float32)[None].copy()
    H[0, 2] = 0.0                     # q2 = 0 for every p0
    assert not G.admissible("fundamental", F, 1e9, p0, p1)[0].any()
    assert not G.admissible("homography", H, 1e9, p0, p1)[0].any()
