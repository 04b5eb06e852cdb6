"""Guided coarse matching (data["guide"], lb_coarse_match_guided; DESIGN.md §18) on the GPU:
1. a guide that admits every entry gives the unguided outputs bit for bit, on every path and option;
2. the guided match lists against the float64 guided reference (ref64.conf_matrix under tests/guided_ref.py's
   admissibility) at the tile, chunk and mask boundaries of tests/test_kernel_edges_gpu.py, with F and H guides whose
   bands cut through the tiles (the near-tie rule of DESIGN.md §5, mconf at rtol 1e-3); cell pairs within 1e-3 r of the
   band's edge are left out;
3. every coarse match lies in the band (recomputed in float64), and conf_matrix is 0 outside it;
4. per-pair behaviour: a NaN model leaves its pair unguided, a pair does not see the other pairs' models, a model that
   maps every cell outside image1 leaves its pair without matches;
5. dual-softmax: a match of both calls has a guided mconf at least its unguided one (rounding aside);
6. forward_static with a guide, captured into a CUDA graph and replayed, equals the eager guided call."""
import numpy as np
import pytest
import torch

import guided_ref as G
import ref64 as R
import util
from cases import CASES, build_cfg, build_cm_inputs
from match_cap_ref import LIST_KEYS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_CASE = {c["name"]: c for c in CASES}
CM_KEYS = ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c")


def _models(kind, n):
    return np.repeat((util.F_MODEL if kind == "fundamental" else util.H_MODEL)[None], n, 0)


def _cm_setup(case, match_type, precision="split", prefilter=False, cap=None, conf=False, scales=False):
    n, (h0, w0), (h1, w1) = case["n"], case["hw0c"], case["hw1c"]
    ot = match_type == "sinkhorn"
    cm_case = {"n": n, "hw0c": (h0, w0), "hw1c": (h1, w1), "amp": 3.0 if ot else 1.6, "frac": 0.6, "iseed": 23}
    if "valid0c" in case:
        cm_case.update(valid0c=case["valid0c"], valid1c=case["valid1c"])
    inp = build_cm_inputs(cm_case)
    mc = build_cfg({"thr": case.get("thr", 0.0), "match_type": match_type, "prefilter": prefilter,
                    "border_rm": case.get("border_rm", 0)})["match_coarse"]
    mc["skh_iters"], mc["dsmax_temperature"] = 3, 0.1
    mc["return_conf_matrix"] = conf
    mc["max_matches_per_pair"] = cap
    import loftr_b200.loftr as LM
    mod = LM.CoarseMatching(mc, precision=precision).eval().to(DEV)
    if ot:
        mod.bin_score.data = torch.tensor(1.0, device=DEV)
    base = {"hw0_i": (h0 * 8, w0 * 8), "hw1_i": (h1 * 8, w1 * 8), "hw0_c": (h0, w0), "hw1_c": (h1, w1)}
    if scales:
        rs = np.random.RandomState(7)
        base["scale0"], base["scale1"] = (util.to_dev(rs.uniform(0.7, 1.6, (n, 2)).astype(np.float32))
                                          for _ in range(2))
    m0 = m1 = None
    if "mask0" in inp:
        base["mask0"], base["mask1"] = util.to_dev(inp["mask0"]), util.to_dev(inp["mask1"])
        m0, m1 = base["mask0"].flatten(-2), base["mask1"].flatten(-2)

    def run(guide=None):
        data = dict(base)
        if guide is not None:
            data["guide"] = guide
        mod(util.to_dev(inp["feat_c0"]), util.to_dev(inp["feat_c1"]), data, m0, m1)
        return data
    return run, inp, mc, base


def _points(case, base):
    n = case["n"]
    s0 = util.to_np(base["scale0"]) if "scale0" in base else None
    s1 = util.to_np(base["scale1"]) if "scale1" in base else None
    return G.coarse_points(n, case["hw0c"], 8.0, s0), G.coarse_points(n, case["hw1c"], 8.0, s1)


# ------------------------------------------------------------------------------------------------ 1. identity
IDENTITY = [pytest.param(mt, prec, pre, masked, cap, id=f"{mt}_{prec}_{'pre' if pre else 'nopre'}_"
                         f"{'masked_scaled' if masked else 'plain'}_cap{cap}")
            for mt, pre in (("dual_softmax", False), ("sinkhorn", False), ("sinkhorn", True))
            for prec in ("split", "fp16") for masked in (False, True) for cap in (None, 7)]


@pytest.mark.parametrize("match_type, precision, prefilter, masked, cap", IDENTITY)
def test_all_admissible_guide_is_bitwise_unguided(match_type, precision, prefilter, masked, cap):
    case = {"n": 3, "hw0c": (12, 11), "hw1c": (10, 27), "border_rm": 1}
    if masked:
        case.update(valid0c=[(12, 11), (9, 8), (12, 6)], valid1c=[(7, 27), (10, 27), (10, 20)])
    run, _, _, _ = _cm_setup(case, match_type, precision, prefilter, cap, conf=True, scales=masked)
    ref = run()
    assert ref["b_ids"].numel() > 0
    rs = np.random.RandomState(1)
    for label, guide in (("radius_1e9_F", util.guide("fundamental", rs.standard_normal((3, 3, 3)), 1e9)),
                         ("radius_1e9_H", util.guide("homography", _models("homography", 3), 1e9)),
                         ("nan_model", util.guide("homography", np.full((3, 3, 3), np.nan), 2.0))):
        got = run(guide)
        util.assert_same(got, ref, CM_KEYS + ("conf_matrix",), label, nan_equal=False)


def _e2e_identity_guides(n):
    return [util.guide("homography", np.repeat(util.H_MODEL[None], n, 0), 1e9),
            util.guide("fundamental", np.full((n, 3, 3), np.nan), 4.0)]


@pytest.mark.parametrize("name", ["ds_thr0", "ds_masked_scaled", "ot_thr0"])
def test_all_admissible_guide_end_to_end_is_bitwise_unguided(name):
    """forward, forward_static and match_features (with estimate=) through the guided entry point."""
    case = _CASE[name]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    ref = util.eager(model, inp)
    n = case["n"]
    for guide in _e2e_identity_guides(n):
        got = util.eager(model, dict(inp, guide=guide))
        util.assert_same(got, ref, LIST_KEYS, "forward", nan_equal=False)
        st = dict(inp, guide=guide)
        model.forward_static(st)
        util.assert_static_equals_eager(st, ref, "forward_static")   # the live prefix of its capacity buffers
    if "mask0" in inp:
        return
    imgs = torch.cat([inp["image0"], inp["image1"]])
    bank = model.extract_features(imgs)
    i0 = torch.arange(n, device=DEV)
    i1 = i0 + n
    ref_mf = model.match_features(bank, i0, bank, i1, estimate="fundamental")
    for guide in _e2e_identity_guides(n):
        got = model.match_features(bank, i0, bank, i1, estimate="fundamental", guide=guide)
        util.assert_same(got, ref_mf, (*LIST_KEYS, "geom_model", "geom_inliers", "geom_num_inliers"), "match_features",
                         nan_equal=False)
        assert "guide" not in got


# ------------------------------------------------------------------------------------------------ 2. against float64
def _cp(cid, **kw):
    return pytest.param(kw, id=cid)


_GRID = {127: (1, 127), 128: (8, 16), 129: (3, 43), 255: (15, 17), 256: (16, 16), 257: (1, 257)}
F64_SHAPES = [_cp(f"L{L}_S{S}", n=3, hw0c=_GRID[L], hw1c=_GRID[S]) for L, S in ((127, 255), (128, 256), (129, 257))] + [
    _cp("multi_chunk_unequal", n=2, hw0c=(12, 20), hw1c=(40, 60), border_rm=2),
    _cp("unequal_48", n=4, hw0c=(6, 8), hw1c=(8, 6)),
    _cp("masked", n=3, hw0c=(12, 16), hw1c=(12, 16), border_rm=2,
        valid0c=[(12, 16), (12, 9), (7, 16)], valid1c=[(10, 16), (9, 16), (12, 11)]),
]
# radii in image pixels (8 per cell): a few cells wide, so the band cuts through every 32 x 32 block and 128-row tile
KINDS = [pytest.param("fundamental", 12.0, id="F_r12"), pytest.param("homography", 28.0, id="H_r28")]


def _vs_f64(case, match_type, kind, radius, precision="split", prefilter=False):
    run, inp, mc, base = _cm_setup(case, match_type, precision, prefilter, conf=True)
    n = case["n"]
    models = _models(kind, n)
    if case["hw0c"][0] == 1 or case["hw1c"][0] == 1:   # one-row grids: a translation keeps the band on the grid
        models = np.repeat(np.array([[1, 0, 40.0], [0, 1, 0], [0, 0, 1]], np.float32)[None], n, 0)
        if kind == "fundamental":
            models = np.repeat(np.array([[0, 0, 0.01], [0, 0, -1], [-0.01, 1, 0]], np.float32)[None], n, 0)
    got = run(util.guide(kind, models, radius))
    p0, p1 = _points(case, base)
    adm, margin = G.admissible(kind, models, radius, p0, p1)
    assert 0.005 < adm.mean() < 0.9, adm.mean()
    m0 = m1 = None
    if "mask0" in base:
        m0, m1 = base["mask0"].flatten(-2), base["mask1"].flatten(-2)
    conf = R.conf_matrix(R.f64(inp["feat_c0"], DEV), R.f64(inp["feat_c1"], DEV), mc, m0, m1, 1.0,
                         fp16=precision == "fp16", adm=util.to_dev(adm))
    ref = R.coarse_match(conf, mc, base["hw0_i"], case["hw0c"], case["hw1c"], base.get("mask0"), base.get("mask1"))
    ref = {k: util.to_np(v) for k, v in ref.items()}
    g = {k: util.to_np(got[k]) for k in CM_KEYS}
    near = margin < 1e-3 * radius

    def drop(d):
        keep = ~near[d["b_ids"], d["i_ids"], d["j_ids"]]
        return {k: v[keep] for k, v in d.items()}
    rows, cols = R.top2(conf)
    gold = {"row_top2_f64": util.to_np(rows), "col_top2_f64": util.to_np(cols)}
    stats = util.compare_matches(drop(g), drop(ref), gold,
                                 conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995, label=f"guided_{match_type}_{kind}")
    assert stats["n"] > 0
    util.record(f"guided_vs_f64_{match_type}_{precision}_{kind}", {**stats, "admissible": float(adm.mean()),
                                                                   "near_boundary": int(near.sum())})
    return got, adm, conf


@pytest.mark.parametrize("kind, radius", KINDS)
@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
@pytest.mark.parametrize("case", F64_SHAPES)
def test_guided_matching_vs_f64(case, match_type, kind, radius):
    _vs_f64(case, match_type, kind, radius, prefilter=match_type == "sinkhorn")


@pytest.mark.parametrize("kind, radius", KINDS)
@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
def test_guided_fp16_vs_f64_emulation(match_type, kind, radius):
    case = {"n": 2, "hw0c": (12, 20), "hw1c": (40, 60), "border_rm": 2}
    _vs_f64(case, match_type, kind, radius, precision="fp16")


# ------------------------------------------------------------------------------------------------ 3. band holds
@pytest.mark.parametrize("kind, radius", KINDS)
@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
def test_matches_lie_in_the_band_and_conf_matrix_is_zero_outside(match_type, kind, radius):
    case = {"n": 2, "hw0c": (12, 20), "hw1c": (14, 18), "border_rm": 1}
    run, _, _, base = _cm_setup(case, match_type, scales=True, conf=True)
    models = _models(kind, 2).astype(np.float64)
    got = run(util.guide(kind, models, radius))
    b = util.to_np(got["b_ids"])
    assert len(b) > 0
    p0, p1 = util.to_np(got["mkpts0_c"]).astype(np.float64), util.to_np(got["mkpts1_c"]).astype(np.float64)
    T = models[b]
    v = np.einsum("mij,mj->mi", T, np.concatenate([p0, np.ones((len(b), 1))], 1))
    if kind == "fundamental":
        dist = np.abs(v[:, 0] * p1[:, 0] + v[:, 1] * p1[:, 1] + v[:, 2]) / np.hypot(v[:, 0], v[:, 1])
    else:
        dist = np.hypot(v[:, 0] / v[:, 2] - p1[:, 0], v[:, 1] / v[:, 2] - p1[:, 1])
    assert dist.max() <= radius * (1 + 1e-5) + 1e-3, dist.max()
    q0, q1 = _points(case, base)
    adm, _ = G.admissible(kind, models, radius, q0, q1)
    cm = util.to_np(got["conf_matrix"])
    assert (cm[~adm] == 0).all() and (cm[adm] > 0).any()


# ------------------------------------------------------------------------------------------------ 4. per pair
@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
def test_per_pair_models(match_type):
    case = {"n": 3, "hw0c": (12, 16), "hw1c": (12, 16), "border_rm": 1}
    run, _, _, _ = _cm_setup(case, match_type, conf=True)
    unguided = run()

    def pair(d, p):
        sel = d["b_ids"] == p
        return {k: d[k][sel] for k in CM_KEYS} | {"conf_matrix": d["conf_matrix"][p]}
    models = _models("homography", 3).copy()
    models[1] = np.nan
    models[2] = [[1, 0, 1e5], [0, 1, 1e5], [0, 0, 1]]     # every cell maps far outside image1
    got = run(util.guide("homography", models, 20.0))
    util.assert_same(pair(got, 1), pair(unguided, 1), CM_KEYS + ("conf_matrix",), "NaN model", nan_equal=False)
    assert not (got["b_ids"] == 2).any() and (got["conf_matrix"][2] == 0).all()
    assert (got["b_ids"] == 0).any()
    for k in ("mconf", "mkpts0_c", "mkpts1_c", "conf_matrix"):
        assert torch.isfinite(got[k]).all(), k
    other = models.copy()
    other[1] = util.H_MODEL                                # change the other pairs' models only
    other[2] = [[0.9, 0.1, -8.0], [0.0, 1.1, 3.0], [0, 0, 1]]
    got2 = run(util.guide("homography", other, 20.0))
    util.assert_same(pair(got2, 0), pair(got, 0), CM_KEYS + ("conf_matrix",), "independent pairs", nan_equal=False)


# ------------------------------------------------------------------------------------------------ 5. monotone mconf
@pytest.mark.parametrize("kind, radius", KINDS)
def test_dual_softmax_confidence_grows_under_a_guide(kind, radius):
    case = {"n": 3, "hw0c": (16, 20), "hw1c": (15, 21), "border_rm": 0}
    run, _, _, _ = _cm_setup(case, "dual_softmax")
    a, g = run(), run(util.guide(kind, _models(kind, 3), radius))
    ka = {k: n for n, k in enumerate(zip(*(util.to_np(a[x]).tolist() for x in ("b_ids", "i_ids", "j_ids"))))}
    kg = {k: n for n, k in enumerate(zip(*(util.to_np(g[x]).tolist() for x in ("b_ids", "i_ids", "j_ids"))))}
    common = sorted(set(ka) & set(kg))
    assert len(common) > 0
    ca, cg = util.to_np(a["mconf"])[[ka[k] for k in common]], util.to_np(g["mconf"])[[kg[k] for k in common]]
    assert (cg >= ca * (1 - 1e-5)).all(), float((cg / ca).min())
    util.record(f"guided_mconf_monotone_{kind}", {"common": len(common), "min_ratio": float((cg / ca).min())})


# ------------------------------------------------------------------------------------------------ 6. graph replay
def test_forward_static_with_guide_replays_from_a_graph():
    case = _CASE["ds_thr0"]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    guide = util.guide("homography", np.repeat(np.eye(3, dtype=np.float32)[None], case["n"], 0), 40.0)
    eager = util.eager(model, dict(inp, guide=guide))
    unguided = util.eager(model, inp)
    assert eager["b_ids"].numel() > 0
    assert eager["b_ids"].shape != unguided["b_ids"].shape or not torch.equal(eager["mconf"], unguided["mconf"])
    st = dict(inp, guide=guide)
    model.forward_static(st)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    out = dict(inp, guide=guide)
    with torch.cuda.graph(g):
        model.forward_static(out)
    g.replay()
    util.assert_static_equals_eager(out, eager, "guided graph replay")
    guide["model"].copy_(torch.full_like(guide["model"], float("nan")))   # the graph reads the model at every replay
    g.replay()
    util.assert_static_equals_eager(out, unguided, "guided graph replay, NaN model")
