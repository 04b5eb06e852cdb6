"""Rectified matching (data["rectify1"], `warp_images`, lb_rectify_images / lb_rectify_points; DESIGN.md §19) on the
GPU:
1. `warp_images` against the float64 grid_sample reference within 4 fp32 ulps of 1.0: canvases that are not a multiple
   of the 128-pixel block row, image1 smaller and larger than the canvas, samples on and just beyond the last row and
   column, horizons crossing the canvas, NaN and negated models next to valid ones, scales;
2. an identity model with equal sizes and scales gives every key of forward, forward_static and match_points bit for
   bit (split and fp16, dual-softmax and Sinkhorn, with a per-pair cap);
3. composition: the rectified call equals the plain call on the substituted input for every key but mkpts1_*, which
   are the float64 back-mapping of the plain call's points within 1 ulp, with minside1 its float64 flag;
4. a pair's outputs do not depend on the other pairs' models;
5. a match_points query at a rectified match's mkpts0_c returns that match's mapped points;
6. forward_static with rectify1 captured into a CUDA graph follows the model tensor from replay to replay."""
import numpy as np
import pytest
import torch

import loftr_b200
import rectify_ref as RR
import util
from cases import CASES
from match_cap_ref import LIST_KEYS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_CASE = {c["name"]: c for c in CASES}
INPUTS = util.INPUT_KEYS + ("rectify1",)
ULP1 = 4 * float(np.finfo(np.float32).eps)   # 4 fp32 ulps of 1.0


def _centre(hw, s=(1.0, 1.0)):
    return (0.5 * (hw[1] - 1) * s[0], 0.5 * (hw[0] - 1) * s[1])


# ------------------------------------------------------------------------------------------------ 1. the warp
def _warp_case(name):
    rs = np.random.RandomState(11)
    if name == "canvas200_scaled":
        n, hw1, hw = 3, (40, 56), (48, 200)
        s0, s1 = rs.uniform(0.6, 1.4, (n, 2)), rs.uniform(0.6, 1.4, (n, 2))
        models = [util.similarity(_centre(hw, s0[b]), _centre(hw1, s1[b]), deg, zoom, persp)
                  for b, (deg, zoom, persp) in enumerate(((7, 0.3, (1e-4, -2e-4)), (-20, 0.25, (0, 0)),
                                                           (90, 0.35, (-3e-4, 1e-4))))]
    elif name == "image1_smaller":
        n, hw1, hw, s0, s1 = 2, (24, 32), (64, 96), None, None
        models = [util.similarity(_centre(hw), _centre(hw1), 3, 0.45),
                  util.similarity(_centre(hw), (30.0, 20.0), -12, 0.5)]
    elif name == "image1_larger":
        n, hw1, hw, s0, s1 = 2, (96, 136), (40, 48), None, None
        models = [util.similarity(_centre(hw), _centre(hw1), 30, 2.5),
                  util.similarity(_centre(hw), _centre(hw1), 180, 2.9)]
    elif name == "edges":   # samples on the last row / column, a quarter pixel beyond it, and before the first
        n, hw1, hw, s0, s1 = 4, (32, 40), (32, 40), None, None
        models = [np.array([[1, 0, tx], [0, 1, ty], [0, 0, 1]], np.float64)
                  for tx, ty in ((0.25, 0.5), (-0.75, 0.0), (1.0, 1.0), (0.0, 0.0))]
    elif name == "horizon_nan_negated":
        n, hw1, hw, s0, s1 = 3, (48, 64), (48, 128), None, None
        models = [np.array([[1, 0, 0], [0, 1, 0], [-0.012, 0, 1.0]]),   # w = 0 at x = 83: the horizon crosses
                  np.full((3, 3), np.nan),
                  -util.similarity(_centre(hw), _centre(hw1), 15, 0.6, (2e-3, 0))]
    else:
        raise KeyError(name)
    img = rs.rand(n, 1, *hw1).astype(np.float32)
    scale0 = None if s0 is None else s0.astype(np.float32)
    scale1 = None if s1 is None else s1.astype(np.float32)
    return img, np.stack(models).astype(np.float32), hw, scale0, scale1


WARP_CASES = ["canvas200_scaled", "image1_smaller", "image1_larger", "edges", "horizon_nan_negated"]


@pytest.mark.parametrize("name", WARP_CASES)
def test_warp_images_vs_float64(name):
    img, models, hw, s0, s1 = _warp_case(name)
    got = loftr_b200.warp_images(util.to_dev(img), util.to_dev(models), hw, None if s0 is None else util.to_dev(s0),
                                 None if s1 is None else util.to_dev(s1))
    torch.cuda.synchronize()
    assert got.shape == (img.shape[0], 1, *hw) and got.dtype == torch.float32
    ref, u, v = RR.warp(img, models, hw, s0, s1)
    keep = ~RR.near_pixel_boundary(u, v)
    err = (got.cpu().double() - ref)[:, 0][keep].abs()
    assert err.max() <= ULP1, (name, float(err.max()))
    h1, w1 = img.shape[2:]
    outside = ~((u > -1) & (u < w1) & (v > -1) & (v < h1))   # no tap in image1, or beyond the horizon (NaN)
    assert (outside.any() or name == "edges") and (~outside).any()
    assert torch.isnan(u).any() == (name == "horizon_nan_negated")
    util.record(f"rectify_warp_{name}", {"max_err": float(err.max()), "kept": int(keep.sum()),
                                         "beyond_horizon": int(torch.isnan(u).sum())})
    g = got.cpu()
    if name == "edges":   # integer shift and identity: exact
        assert torch.equal(g[2, 0, :-1, :-1], torch.from_numpy(img[2, 0, 1:, 1:]))
        assert (g[2, 0, -1] == 0).all() and (g[2, 0, :, -1] == 0).all()
        assert torch.equal(g[3], torch.from_numpy(img[3]))
    if name == "horizon_nan_negated":   # the NaN model is the identity: image1 top-left, zeros right of it
        assert torch.equal(g[1, :, :, :64], torch.from_numpy(img[1])) and (g[1, :, :, 64:] == 0).all()
        assert (g[0, 0, :, 84:] == 0).all()


def test_warp_images_is_bitwise_image1_for_the_identity_with_scales():
    rs = np.random.RandomState(2)
    img = rs.rand(3, 1, 48, 72).astype(np.float32)
    s = util.to_dev(rs.uniform(0.5, 2.5, (3, 2)), torch.float32)
    models = util.to_dev(np.stack([np.eye(3), np.full((3, 3), np.inf), -np.eye(3)]), torch.float32)
    got = loftr_b200.warp_images(util.to_dev(img), models, (48, 72), s, s.clone())
    assert torch.equal(got.cpu(), torch.from_numpy(img))


# ------------------------------------------------------------------------------------------------ 2. identity
IDENTITY = [("ds_thr0", "split", None), ("ds_thr0", "fp16", None), ("ot_thr0", "split", None),
            ("ds_masked_scaled", "split", 7), ("ot_masked", "fp16", 5)]


def _equalised(case):
    """The case's inputs with image1's scale and mask set to image0's, so that an identity model is a plain copy."""
    inp = util.device_inputs(case)
    if "scale0" in inp:
        inp["scale1"] = inp["scale0"].clone()
    if "mask0" in inp:
        inp["mask1"] = inp["mask0"].clone()
    return inp


def _query_points(data, extra=64, seed=0):
    """Every cell keypoint of image0 (as the forward computes mkpts0_c) and `extra` random points, some outside."""
    n, _, h, w = data["image0"].shape
    s = 8.0 * data["scale0"][:, None, :] if "scale0" in data else torch.full((n, 1, 2), 8.0, device=DEV)
    g = torch.Generator().manual_seed(seed)
    rnd = (torch.rand(n, extra, 2, generator=g) * 1.2 - 0.1).to(DEV) * torch.tensor([w, h], device=DEV) * s / 8.0
    return torch.cat([util.grid_points(data), rnd], 1).contiguous()


@pytest.mark.parametrize("name, precision, cap", IDENTITY, ids=[f"{a}_{b}_cap{c}" for a, b, c in IDENTITY])
def test_identity_model_is_bitwise_the_plain_call(name, precision, cap):
    case = _CASE[name]
    model, _, _ = util.build_model(case, DEV, match_precision=precision)
    model.coarse_matching.max_matches_per_pair = cap
    inp = _equalised(case)
    n = inp["image0"].shape[0]
    eye = torch.eye(3, device=DEV).repeat(n, 1, 1)
    ref = util.eager(model, inp)
    assert ref["b_ids"].numel() > 0
    for label, rect in (("identity", eye), ("nan", torch.full_like(eye, float("nan"))), ("negated", -eye)):
        got = util.eager(model, dict(inp, rectify1=rect))
        util.assert_same(got, util.outputs(ref, INPUTS), label=f"forward {label}")
        assert got["minside1"].dtype == torch.bool and got["minside1"].shape == ref["b_ids"].shape
        want = RR.map_back(ref["mkpts1_f"], ref["m_bids"], eye, inp["image0"].shape[2:], inp["image1"].shape[2:],
                           inp.get("scale0"), inp.get("scale1"), inp.get("mask1"))[1]
        assert torch.equal(got["minside1"].cpu(), want), label
        for k in ("image1", "rectify1"):
            assert got[k] is (inp[k] if k in inp else rect)
    st = dict(inp, rectify1=eye)
    model.forward_static(st)
    util.assert_static_equals_eager(st, ref, "forward_static identity")
    pts = _query_points(inp)
    qref, qgot = dict(inp), dict(inp, rectify1=eye)
    model.match_points(qref, pts)
    model.match_points(qgot, pts)
    util.assert_same(qgot, util.outputs(qref, INPUTS), label="match_points identity")
    assert qgot["qinside1"].shape == qref["qinside"].shape


# ------------------------------------------------------------------------------------------------ 3. composition
def _models_for(inp, seed):
    """A mild homography per pair about the image centres, in source pixels (rotation, zoom and perspective)."""
    rs = np.random.RandomState(seed)
    n, hw0, hw1 = inp["image0"].shape[0], inp["image0"].shape[2:], inp["image1"].shape[2:]
    s0 = inp["scale0"].cpu().numpy() if "scale0" in inp else np.ones((n, 2))
    s1 = inp["scale1"].cpu().numpy() if "scale1" in inp else np.ones((n, 2))
    m = [util.similarity(_centre(hw0, s0[b]), _centre(hw1, s1[b]), rs.uniform(-25, 25), rs.uniform(0.8, 1.25),
                     rs.uniform(-4e-4, 4e-4, 2) / max(s0[b])) for b in range(n)]
    return util.to_dev(np.stack(m), torch.float32)


def _substituted(inp, rect):
    sub = {"image0": inp["image0"],
           "image1": loftr_b200.warp_images(inp["image1"], rect, inp["image0"].shape[2:], inp.get("scale0"),
                                            inp.get("scale1"))}
    if "scale0" in inp:
        sub["scale0"] = sub["scale1"] = inp["scale0"]
    if "mask0" in inp:
        sub["mask0"] = sub["mask1"] = inp["mask0"]
    return sub


def _assert_mapped(got, ref_pts, ref_ids, rect, inp, label, key_pts, key_inside):
    want, want_in = RR.map_back(ref_pts, ref_ids, rect, inp["image0"].shape[2:], inp["image1"].shape[2:],
                                inp.get("scale0"), inp.get("scale1"), inp.get("mask1"))
    g = got[key_pts].reshape(-1, 2).cpu().double()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(g), nan), label
    ulp = torch.from_numpy(np.spacing(np.abs(want[~nan].numpy()).astype(np.float32)).astype(np.float64))
    assert ((g[~nan] - want[~nan]).abs() <= ulp).all(), f"{label}: {key_pts} beyond 1 ulp"
    if key_inside is not None:
        assert torch.equal(got[key_inside].reshape(-1).cpu(), want_in), f"{label}: {key_inside}"
        return want_in


@pytest.mark.parametrize("name", ["ds_thr0", "ds_masked_scaled", "ot_masked", "ds_unequal"])
def test_rectified_call_is_the_plain_call_on_the_substituted_input(name):
    case = _CASE[name]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    rect = _models_for(inp, 5)
    got = util.eager(model, dict(inp, rectify1=rect))
    plain = util.eager(model, _substituted(inp, rect))
    assert plain["b_ids"].numel() > 0
    util.assert_same(got, plain, [k for k in util.outputs(plain, INPUTS) if k not in ("mkpts1_c", "mkpts1_f")], name)
    _assert_mapped(got, plain["mkpts1_c"], plain["m_bids"], rect, inp, name, "mkpts1_c", None)
    flags = _assert_mapped(got, plain["mkpts1_f"], plain["m_bids"], rect, inp, name, "mkpts1_f", "minside1")
    util.record(f"rectify_composition_{name}", {"matches": int(plain["b_ids"].numel()), "inside": int(flags.sum())})
    pts = _query_points(inp, seed=3)
    qgot, qplain = dict(inp, rectify1=rect), _substituted(inp, rect)
    model.match_points(qgot, pts)
    model.match_points(qplain, pts)
    n, q = pts.shape[:2]
    util.assert_same(qgot, qplain, [k for k in util.outputs(qplain, INPUTS) if k not in ("qpts1_c", "qpts1_f")],
                     f"{name} points")
    ids = torch.arange(n).repeat_interleave(q)
    _assert_mapped(qgot, qplain["qpts1_c"].reshape(-1, 2), ids, rect, inp, f"{name} points", "qpts1_c", None)
    _assert_mapped(qgot, qplain["qpts1_f"].reshape(-1, 2), ids, rect, inp, f"{name} points", "qpts1_f", "qinside1")


# ------------------------------------------------------------------------------------------------ 4. per pair
def test_pairs_do_not_see_the_other_pairs_models():
    case = _CASE["ds_thr0"]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    a = _models_for(inp, 7)
    b = a.clone()
    b[1] = _models_for(inp, 8)[1]
    ra, rb = util.eager(model, dict(inp, rectify1=a)), util.eager(model, dict(inp, rectify1=b))
    sa, sb = ra["b_ids"] == 0, rb["b_ids"] == 0
    assert sa.any()
    keys = LIST_KEYS + ["minside1"]
    util.assert_same({k: ra[k][sa] for k in keys}, {k: rb[k][sb] for k in keys}, label="pair 0")
    assert not util.same(ra["mkpts1_f"][~sa], rb["mkpts1_f"][~sb])


# ------------------------------------------------------------------------------------------------ 5. point queries
@pytest.mark.parametrize("name", ["ds_thr0", "ds_masked_scaled"])
def test_query_at_a_rectified_match_returns_its_mapped_points(name):
    case = _CASE[name]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    rect = _models_for(inp, 9)
    fwd = util.eager(model, dict(inp, rectify1=rect))
    n = inp["image0"].shape[0]
    b = fwd["b_ids"]
    counts = torch.bincount(b, minlength=n).tolist()
    q = max(counts)
    assert q > 0
    pts = torch.zeros(n, q, 2, device=DEV)
    valid = torch.zeros(n, q, dtype=torch.bool, device=DEV)
    slot = torch.cat([torch.arange(c, device=DEV) for c in counts])
    pts[b, slot], valid[b, slot] = fwd["mkpts0_c"], True
    out = dict(inp, rectify1=rect)
    model.match_points(out, pts, valid)
    for qk, fk in (("qpts1_c", "mkpts1_c"), ("qpts1_f", "mkpts1_f"), ("qinside1", "minside1"), ("q_j_ids", "j_ids"),
                   ("qconf", "mconf"), ("qexpec_f", "expec_f")):
        util.assert_same(out[qk][b, slot], fwd[fk], label=qk)


# ------------------------------------------------------------------------------------------------ 6. graph replay
def test_forward_static_with_rectify1_replays_from_a_graph():
    case = _CASE["ds_masked_scaled"]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    m1, m2 = _models_for(inp, 1), _models_for(inp, 2)
    e1, e2 = util.eager(model, dict(inp, rectify1=m1)), util.eager(model, dict(inp, rectify1=m2))
    assert e1["b_ids"].numel() > 0 and not util.same(e1["mkpts1_f"], e2["mkpts1_f"])
    rect = m1.clone()
    model.forward_static(dict(inp, rectify1=rect))   # eager warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    out = dict(inp, rectify1=rect)
    with torch.cuda.graph(g):
        model.forward_static(out)
    for label, m, eager in (("model 1", m1, e1), ("model 2", m2, e2)):
        rect.copy_(m)   # the graph reads the model from the same tensor at every replay
        g.replay()
        util.assert_static_equals_eager(out, eager, f"rectified graph replay, {label}")
        k = int(out["num_matches"].item())
        assert torch.equal(out["minside1"][:k], eager["minside1"]), label
