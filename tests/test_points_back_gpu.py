"""Image1-side point queries and round trips on the GPU (DESIGN.md §22):
1. an image1 query at every cell keypoint mirrors the forward: at each match's mkpts1_c it returns the match's ids,
   mconf and flags bit for bit, with the forward's windows; qmutual / qvalid / the mutual qconf are the image0-side
   answers of the same cell pair (split and fp16, dual-softmax and Sinkhorn with and without the prefilter, linear and
   full attention, 832 x 832 masks and scales);
2. off-grid image1 queries against float64 (tests/points_ref.py): the column arg-max, both qconf expressions, the
   centres and the mirrored fine match on the stored stage inputs, at the image edges and window borders; masked cells
   and columns without a valid row are not answered;
3. the back leg of a round trip equals a separate call from the other image at the first answer, from both sides,
   stacked and on banks, with a guide and an all-NaN guide; the back leg runs no score pass;
4. image1 queries and round trips on banks equal the stacked calls bit for bit;
5. a round trip leaves the first leg's outputs as a call without it computes them;
6. a captured round trip replays equal to the eager call."""
import numpy as np
import pytest
import torch

from loftr_b200 import _lib
import points_ref as P
import ref64 as R
import util
from cases import BASELINE_CASES, CASES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASE = {c["name"]: c for c in CASES}
BACK = ("qback_pts", "qback_conf", "qback_valid", "qback_inside", "qfb_err")


def _query(model, data, side, pts, valid=None, **kw):
    out = util.inputs(data)
    model.match_points(out, **{f"points{side}": pts, f"valid{side}": valid}, **kw)
    return util.outputs(out)


def _offgrid_points(n, h, w, seed, q=150):
    """Image corners and edges (windows partly outside the fine map), the last cell row and column, and sub-pixel
    points -> [n, Q, 2]."""
    rs = np.random.RandomState(seed)
    edges = [(0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1), (0.4, h / 3), (w - 1.2, 21.7), (w / 2 + .49, 0.3),
             (29.1, h - 1.4), (w - 4.6, h - 4.6), (w - 9.0, h - 9.0), (3.9, 4.1), (w / 2 + 0.49, h / 2 + 1.51)]
    pts = [np.concatenate([np.asarray(edges, np.float64), np.stack([rs.uniform(0, w - 1, q), rs.uniform(0, h - 1, q)],
                                                                   1)]) for _ in range(n)]
    return torch.tensor(np.stack(pts), dtype=torch.float32, device=DEV)


# ------------------------------------------------------------------------------------------------ 1. mirror
GRID = [
    ("ds_thr0_border2", CASE["ds_thr0"], {}),
    ("out4_masked_scaled", BASELINE_CASES["out4"], {}),
    ("ds_unequal", CASE["ds_unequal"], {}),
    ("ot_thr0", CASE["ot_thr0"], {}),
    ("ot_prefilter", CASE["ot_prefilter"], {}),
    ("full_attention", dict(CASE["ds_thr0"], coarse_attention="full", fine_attention="full"), {}),
    ("fp16", CASE["ds_thr0"], {"backbone_impl": "b200_fp16", "match_precision": "fp16"}),
    ("ot_fp16", CASE["ot_thr0"], {"match_precision": "fp16"}),
]


@pytest.mark.parametrize("name, case, opts", GRID, ids=[g[0] for g in GRID])
def test_image1_grid_queries_mirror_the_forward(name, case, opts):
    model, _, _ = util.build_model(case, DEV, **opts)
    data = util.device_inputs(case)
    fwd = util.eager(model, data)
    q = _query(model, data, 1, util.grid_points(data, 1))
    q0 = _query(model, data, 0, util.grid_points(data, 0))   # the image0 side of every cell pair
    n, S = q["qvalid"].shape
    b, i, j = fwd["b_ids"], fwd["i_ids"], fwd["j_ids"]
    if name == "ot_prefilter":   # the prefilter removes every row and column of this pair: nothing is kept or valid
        assert len(b) == 0 and not q["qvalid"].any()
    else:
        assert len(b) > 0, name
        assert q["qinside"][b, j].all() and q["qvalid"][b, j].all() and q["qmutual"][b, j].all(), name
        for qk, fk in (("q_i_ids", "i_ids"), ("q_j_ids", "j_ids"), ("qconf", "mconf"), ("qpts1_f", "mkpts1_c"),
                       ("qpts0_c", "mkpts0_c")):
            assert torch.equal(q[qk][b, j], fwd[fk]), f"{name}: {qk} differs from the forward's {fk}"
        others = torch.ones(n, S, dtype=torch.bool, device=DEV)
        others[b, j] = False
        assert not q["qvalid"][others].any(), f"{name}: a cell the forward drops has qvalid"
    assert not (q["qvalid"] & ~q["qmutual"]).any() and not (q["qmutual"] & ~q["qinside"]).any()
    if "mask1" in data:
        assert not q["qinside"][~data["mask1"].reshape(n, S)].any()
    # mutual, valid and the mutual conf are the image0 side's answers for row i
    bb, jj = torch.nonzero(q["qinside"], as_tuple=True)
    ii = q["q_i_ids"][bb, jj]
    mutual = q0["q_j_ids"][bb, ii] == jj
    assert torch.equal(q["qmutual"][bb, jj], mutual) and torch.equal(q["qvalid"][bb, jj], mutual & q0["qvalid"][bb, ii])
    assert torch.equal(q["qconf"][bb, jj][mutual], q0["qconf"][bb, ii][mutual])
    util.record(f"points_back_grid_{name}", {"matches": int(len(b)), "answered": int(len(bb)),
                                             "mutual": int(mutual.sum())})


# ------------------------------------------------------------------------------------------------ 2. vs float64
def _stage_inputs(model, data):
    """The kernel's own stage inputs of `data`: fine maps and coarse transformer outputs."""
    model.expose_coarse_features = True
    fwd = util.eager(model, data)
    model.expose_coarse_features = False
    n = data["image0"].shape[0]
    with torch.no_grad():
        if data["image0"].shape == data["image1"].shape:
            _, ff = model._backbone(torch.cat([data["image0"], data["image1"]]))
            ff0, ff1 = ff[:n], ff[n:]
        else:
            (_, ff0), (_, ff1) = model._backbone(data["image0"]), model._backbone(data["image1"])
    return fwd, ff0, ff1, fwd["_feat_c0"], fwd["_feat_c1"]


QCONF_RTOL = 1e-3   # |qconf - conf64| / conf64, both expressions (DESIGN.md §22)


@pytest.mark.parametrize("name", ["ds_thr0", "ds_unequal", "ot_thr0"])
def test_image1_offgrid_queries_vs_f64(name):
    case = CASE[name]
    model, cfg, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    n, _, h1, w1 = data["image1"].shape
    pts = _offgrid_points(n, h1, w1, 5)
    q = _query(model, data, 1, pts)
    assert q["qinside"].all()
    fwd, ff0, ff1, x0, x1 = _stage_inputs(model, data)
    hw0_i, (h0c, w0c), hw1_i, hw1_c, hw1_f = fwd["hw0_i"], fwd["hw0_c"], fwd["hw1_i"], fwd["hw1_c"], fwd["hw1_f"]
    stride = hw1_f[0] // hw1_c[0]
    mc = cfg["match_coarse"]
    bin_score = model.coarse_matching.bin_score.detach().double() if mc["match_type"] == "sinkhorn" else None
    conf64 = R.conf_matrix(R.f64(x0, DEV), R.f64(x1, DEV), mc, bin_score=bin_score)
    nq = pts.shape[1]
    b_ids = torch.arange(n, device=DEV)[:, None].expand(-1, nq).reshape(-1)
    i_ids, j_ids = q["q_i_ids"].reshape(-1), q["q_j_ids"].reshape(-1)
    # rules 1 and 2 on image1: image0's with image1's sizes
    cells, f1s = [], []
    for b in range(n):
        inside, cell, f1 = P.query_cells(pts[b].cpu().numpy(), None, hw1_i, hw1_c, hw1_f)
        assert inside.all()
        cells.append(cell)
        f1s.append(f1)
    cell, f1 = np.concatenate(cells), np.concatenate(f1s)
    assert (cell[:, 1] * hw1_c[1] + cell[:, 0] == j_ids.cpu().numpy()).all()
    # rule 3: i against the float64 column arg-max, near-ties excepted; qconf within QCONF_RTOL of conf64[b, i, j]
    i64, _, _ = P.column_answer(conf64, b_ids, j_ids)
    cols = conf64[b_ids, :, j_ids]
    top = cols.topk(2, dim=1).values
    for k in torch.nonzero(i64 != i_ids).flatten().tolist():
        gap = ((top[k, 0] - top[k, 1]) / top[k, 0].clamp(min=1e-30)).item()
        assert gap < 1e-2, f"query {k}: i {int(i_ids[k])} vs f64 {int(i64[k])}"
    c64 = conf64[b_ids, i_ids, j_ids]
    rel = ((q["qconf"].reshape(-1).double() - c64).abs() / c64).cpu()
    mutual = q["qmutual"].reshape(-1).cpu()
    assert mutual.any() and (~mutual).any(), "both qconf expressions must be exercised"
    for label, sel in (("mutual", mutual), ("column", ~mutual)):
        err = rel[sel].max().item()
        util.record(f"points_back_qconf_{name}_{label}", {"max_rel_err": err, "queries": int(sel.sum())})
        assert err <= QCONF_RTOL, f"{label} qconf: relative error {err:.3e}"
    # rule 4: the centres, image0's rule with the images swapped
    f0 = P.image1_centres(cell, f1, i_ids.cpu().numpy(), w0c, stride)
    assert torch.equal(q["qpts1_f"].reshape(-1, 2).cpu(), torch.tensor(2.0 * f1, dtype=torch.float32))
    assert torch.equal(q["qpts0_c"].reshape(-1, 2).cpu(), torch.tensor(2.0 * f0, dtype=torch.float32))
    # rule 5: the mirrored fine match from the kernel's own cell pairs, against float64 and its float32 emulation
    pts0_c = q["qpts0_c"].reshape(-1, 2)
    refs = {dt: P.fine_stage(model, ff0.to(dt), ff1.to(dt), x0.to(dt), x1.to(dt), b_ids, i_ids, j_ids, f0, f1,
                             pts0_c, hw0_i, dtype=dt, side=1) for dt in (torch.float64, torch.float32)}
    for k, got in (("qexpec_f", q["qexpec_f"].reshape(-1, 3)), ("qpts0_f", q["qpts0_f"].reshape(-1, 2))):
        idx = 0 if k == "qexpec_f" else 1
        ref, emu = refs[torch.float64][idx], refs[torch.float32][idx].double()
        ek, eo = (got.double() - ref).abs().max().item(), (emu - ref).abs().max().item()
        scale = ref.abs().max().item()
        util.record(f"points_back_offgrid_{name}_{k}", {"err_kernel_vs_f64": ek, "err_fp32_vs_f64": eo,
                                                        "scale": scale})
        assert ek <= 4 * eo + 1e-6 * scale, f"{k}: kernel error {ek:.3e} vs fp32 emulation {eo:.3e}"


def _assert_unanswered(q, sel, label):
    for k in ("qpts1_f", "qpts0_c", "qpts0_f", "qexpec_f"):
        assert torch.isnan(q[k][sel]).all(), (label, k)
    assert (q["qconf"][sel] == 0).all() and (q["q_i_ids"][sel] == -1).all() and (q["q_j_ids"][sel] == -1).all()
    for k in ("qmutual", "qvalid", "qinside"):
        assert not q[k][sel].any(), (label, k)


def test_masked_cells_and_columns_without_a_valid_row():
    case = CASE["ds_masked_scaled"]
    model, _, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    n, _, h, w = data["image1"].shape
    pts = (_offgrid_points(n, h, w, 6, q=60) * data["scale1"][:, None]).contiguous()
    valid1 = torch.ones(pts.shape[:2], dtype=torch.bool, device=DEV)
    valid1[:, 3] = False
    q = _query(model, data, 1, pts, valid1)
    s = data["scale1"][:, None]
    cell = torch.clamp(torch.floor(pts / s / 8 + 0.5), min=0).long()
    cell[..., 0].clamp_(max=w // 8 - 1)
    cell[..., 1].clamp_(max=h // 8 - 1)
    unmasked = data["mask1"][torch.arange(n, device=DEV)[:, None], cell[..., 1], cell[..., 0]]
    assert (~unmasked).any() and unmasked.any()
    assert torch.equal(q["qinside"], unmasked & valid1)
    _assert_unanswered(q, ~q["qinside"], "masked")
    data["mask0"][1] = False   # pair 1: every row masked, so no column has a valid row
    q = _query(model, data, 1, pts, valid1)
    assert q["qinside"][0].any()
    _assert_unanswered(q, (slice(1, 2),), "no valid row")


# ------------------------------------------------------------------------------------------------ 3, 5. round trip
def _check_round_trip(call, side, pts, label):
    """call(side, points, valid, round_trip) -> outputs.  The first leg equals a call without the round trip, the back
    leg a call from the other image at the first answer with valid = qinside; qfb_err is the round-trip distance."""
    rt = call(side, pts, None, True)
    plain = call(side, pts, None, False)
    assert set(rt) == set(plain) | set(BACK), label
    util.assert_same(rt, plain, label=f"{label}: first leg")
    other = 1 - side
    back = call(other, rt[f"qpts{other}_f"], rt["qinside"], False)
    for k, ref in (("qback_pts", f"qpts{side}_f"), ("qback_conf", "qconf"), ("qback_valid", "qvalid"),
                   ("qback_inside", "qinside")):
        util.assert_same(rt[k], back[ref], label=f"{label}: {k} against {ref}")
    err = torch.linalg.vector_norm(rt["qback_pts"] - pts, dim=-1).masked_fill_(~rt["qback_inside"], float("nan"))
    util.assert_same(rt["qfb_err"], err, label=f"{label}: qfb_err")
    assert rt["qback_inside"].any() and not (rt["qback_inside"] & ~rt["qinside"]).any(), label
    assert torch.isfinite(rt["qfb_err"][rt["qback_inside"]]).all(), label
    return rt


RT = [("ds_masked_scaled", {}), ("ds_unequal", {}), ("ot_thr0", {"match_precision": "fp16"})]


@pytest.mark.parametrize("name, opts", RT, ids=[r[0] for r in RT])
def test_round_trip_back_leg_equals_a_call_from_the_other_image(name, opts):
    case = CASE[name]
    model, _, _ = util.build_model(case, DEV, **opts)
    data = util.device_inputs(case)
    call = lambda side, pts, valid, rt: _query(model, data, side, pts, valid, round_trip=rt)
    for side in (0, 1):
        n, _, h, w = data[f"image{side}"].shape
        pts = _offgrid_points(n, h, w, 7 + side, q=100)
        if f"scale{side}" in data:
            pts = (pts * data[f"scale{side}"][:, None]).contiguous()
        rt = _check_round_trip(call, side, pts, f"{name} side {side}")
        util.record(f"points_back_round_trip_{name}_{side}", {
            "back_inside": int(rt["qback_inside"].sum()), "median_fb_err": rt["qfb_err"].nanmedian().item()})


def test_the_back_leg_runs_no_score_pass():
    case = CASE["ds_thr0"]
    model, _, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    n, _, h, w = data["image0"].shape
    pts = _offgrid_points(n, h, w, 9, q=40)
    counts = {}
    for rt in (False, True):
        _query(model, data, 0, pts, round_trip=rt)   # warm-up: weight packing
        _lib.timing_enable(True)
        _query(model, data, 0, pts, round_trip=rt)
        torch.cuda.synchronize()
        counts[rt] = _lib.timing_collect()
        _lib.timing_enable(False)
    for tag in ("score_lse", "score_argmax"):
        assert counts[True][tag][1] == counts[False][tag][1] > 0, tag
    assert counts[True]["match_query"][1] == 2 * counts[False]["match_query"][1] == 2
    assert counts[True]["fine_merge"][1] == 2 * counts[False]["fine_merge"][1]


# ------------------------------------------------------------------------------------------------ 3, 4. banks
BANK_MODES = [
    ("ds_b200_split", "ds_thr0", {}),
    ("ds_fp16backbone_fp16match", "ds_thr0", {"backbone_impl": "b200_fp16", "match_precision": "fp16"}),
    ("sinkhorn", "ot_thr0", {}),
    ("masked_scaled", "ds_masked_scaled", {}),
]


@pytest.mark.parametrize("name, case, opts", BANK_MODES, ids=[m[0] for m in BANK_MODES])
def test_bank_image1_queries_and_round_trips_equal_stacked(name, case, opts):
    case = CASE[case]
    model, _, _ = util.build_model(case, DEV, **opts)
    imgs, masks, scales = util.frames(case)
    bank = model.extract_features(imgs, masks)
    idx0, idx1 = util.idx([0, 1, 2, 2]), util.idx([1, 2, 3, 3])
    data = {"image0": imgs[idx0], "image1": imgs[idx1]}
    if masks is not None:
        data["mask0"], data["mask1"] = masks[idx0], masks[idx1]
    if scales is not None:
        data["scale0"], data["scale1"] = scales[idx0], scales[idx1]
    h, w = imgs.shape[2:]
    pts = _offgrid_points(len(idx0), h, w, 10, q=120)
    for side in (0, 1):
        p = pts if scales is None else (pts * scales[(idx0, idx1)[side]][:, None]).contiguous()
        for rt in (False, True):
            got = model.match_points_features(bank, idx0, bank, idx1, scale0=scales, scale1=scales,
                                              **{f"points{side}": p}, round_trip=rt)
            ref = _query(model, data, side, p, round_trip=rt)
            assert set(got) == set(ref), name
            util.assert_same(got, ref, label=f"{name} side {side} round_trip {rt}")
            assert got["qinside"].any()


def test_bank_round_trips_with_a_guide_and_an_all_nan_guide():
    case = CASE["ds_thr0"]
    model, _, _ = util.build_model(case, DEV)
    imgs, _, _ = util.frames(case)
    bank = model.extract_features(imgs)
    idx0, idx1 = util.idx([0, 1, 2, 0]), util.idx([1, 2, 3, 1])
    models = np.repeat(util.H_MODEL[None], 4, 0)
    models[-1] = np.nan   # the last pair repeats the first, unguided
    h, w = imgs.shape[2:]
    pts = _offgrid_points(4, h, w, 11, q=120)
    for guide in (util.guide("homography", models, 20.0), None):
        def call(side, p, valid, rt):
            return model.match_points_features(bank, idx0, bank, idx1, guide=guide, round_trip=rt,
                                               **{f"points{side}": p, f"valid{side}": valid})
        for side in (0, 1):
            _check_round_trip(call, side, pts, f"guide {guide is not None} side {side}")
    nan_guide = util.guide("homography", np.full((4, 3, 3), np.nan), 20.0)
    for side in (0, 1):
        got = model.match_points_features(bank, idx0, bank, idx1, guide=nan_guide, round_trip=True,
                                          **{f"points{side}": pts})
        ref = model.match_points_features(bank, idx0, bank, idx1, round_trip=True, **{f"points{side}": pts})
        util.assert_same(got, ref, label=f"NaN guide side {side}")


# ------------------------------------------------------------------------------------------------ 6. graph capture
def test_graph_capture_of_a_round_trip_replays_the_eager_call():
    case = CASE["ds_masked_scaled"]
    model, _, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    n, _, h, w = data["image1"].shape
    s = data["scale1"][:, None]
    pts_a = (_offgrid_points(n, h, w, 12) * s).contiguous()
    pts_b = (_offgrid_points(n, h, w, 13) * s).contiguous()
    static_in, static_pts = util.inputs(data), pts_a.clone()
    model.match_points(dict(static_in), points1=static_pts, round_trip=True)   # eager warm-up (weight packing)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        model.match_points(dict(static_in), points1=static_pts, round_trip=True)
    torch.cuda.current_stream().wait_stream(stream)
    graph, out = torch.cuda.CUDAGraph(), dict(static_in)
    with torch.cuda.graph(graph):
        model.match_points(out, points1=static_pts, round_trip=True)
    for pts in (pts_b, pts_a):
        static_pts.copy_(pts)
        graph.replay()
        torch.cuda.synchronize()
        ref = _query(model, data, 1, pts, round_trip=True)
        util.assert_same(out, ref, label="graph replay")
