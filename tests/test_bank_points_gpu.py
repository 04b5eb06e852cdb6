"""`LoFTR.match_points_features` on the GPU (point queries on bank pairs, DESIGN.md §21):
1. unguided, it writes what `match_points` writes for the stacked pairs, bit for bit with the tensor-core backbones in
   every mode (backbones, match precisions, dual-softmax and Sinkhorn, linear and full attention, masks and scales at
   832 x 832, a chain with repeated indices, feats1 is feats0, two banks of different sizes); the PyTorch backbone
   follows the match-list rule instead;
2. an all-NaN guide is the unguided call bit for bit;
3. guided grid queries return guided `match_features` matches bit for bit, and qvalid is exactly its match set;
4. every answered guided query's cell pair is admissible (tests/guided_ref.py's bitwise predicate), and a row without
   an admissible column is not answered;
5. guided off-grid queries against float64 (tests/points_ref.py, tests/guided_ref.py and ref64.conf_matrix under the
   guide's admissibility) at the tolerances of §17;
6. a bank tied to stale weights raises."""
import numpy as np
import pytest
import torch

import guided_ref as G
import points_ref as P
import ref64 as R
import util
from cases import BASELINE_CASES, CASES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASE = {c["name"]: c for c in CASES}
Q_KEYS = ("qpts0_f", "qpts1_c", "qpts1_f", "qexpec_f", "qconf", "q_i_ids", "q_j_ids", "qmutual", "qvalid", "qinside")


def _points(idx0, hw, scales, seed, q=160):
    """Cell keypoints, image edges and sub-pixel points of image0 of each pair, in source pixels -> [B, Q, 2]."""
    h, w = hw
    rs = np.random.RandomState(seed)
    b = len(idx0)
    edges = np.array([(0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1), (0.4, h / 3), (w - 1.2, 21.7), (w / 2 + .49, .3),
                      (w - 4.6, h - 4.6), (3.9, 4.1)], np.float64)
    cells = np.stack([rs.randint(0, w // 8, 40), rs.randint(0, h // 8, 40)], 1) * 8.0
    pts = [np.concatenate([edges, cells, np.stack([rs.uniform(0, w - 1, q), rs.uniform(0, h - 1, q)], 1)])
           for _ in range(b)]
    pts = torch.tensor(np.stack(pts), dtype=torch.float32, device=DEV)
    if scales is not None:
        pts = pts * scales[idx0][:, None]
    return pts.contiguous()


def _stacked(model, imgs0, idx0, imgs1, idx1, pts, masks=None, scales=None, valid0=None):
    """match_points on the explicitly stacked pairs -> the keys it wrote."""
    data = {"image0": imgs0[idx0], "image1": imgs1[idx1]}
    if masks is not None:
        data["mask0"], data["mask1"] = masks[0][idx0], masks[1][idx1]
    if scales is not None:
        data["scale0"], data["scale1"] = scales[0][idx0], scales[1][idx1]
    model.match_points(data, pts, valid0)
    return util.outputs(data)


# ------------------------------------------------------------------------------------------------ 1. = stacked
MODES = [
    ("ds_b200_split", "ds_thr0", {}),
    ("ds_b200_fp16match", "ds_thr0", {"match_precision": "fp16"}),
    ("ds_fp16backbone_fp16match", "ds_thr0", {"backbone_impl": "b200_fp16", "match_precision": "fp16"}),
    ("ds_fp16backbone_split", "ds_thr0", {"backbone_impl": "b200_fp16"}),
    ("sinkhorn", "ot_thr0", {}),
    ("sinkhorn_fp16", "ot_thr0", {"match_precision": "fp16"}),
    ("full_attention", "full", {}),
    ("masked_scaled", "ds_masked_scaled", {}),
]


@pytest.mark.parametrize("name, case, opts", MODES, ids=[m[0] for m in MODES])
def test_bank_queries_equal_stacked_match_points_bitwise(name, case, opts):
    case = dict(CASE["ds_thr0"], coarse_attention="full", fine_attention="full") if case == "full" else CASE[case]
    model, _, _ = util.build_model(case, DEV, **opts)
    imgs, masks, scales = util.frames(case)
    bank = model.extract_features(imgs, masks)
    n = case["n"]
    assert n == 2
    # a chain 0 -> 1 -> 2 -> 3 over the bank, a repeated pair and a self pair, in one list; feats1 is feats0
    idx0, idx1 = util.idx([0, 1, 2, 2, 3]), util.idx([1, 2, 3, 3, 3])
    pts = _points(idx0, imgs.shape[2:], scales, 3)
    valid0 = torch.rand(pts.shape[:2], generator=torch.Generator().manual_seed(1)).to(DEV) > 0.1
    for v in (None, valid0):
        got = model.match_points_features(bank, idx0, bank, idx1, pts, v, scales, scales)
        ref = _stacked(model, imgs, idx0, imgs, idx1, pts, None if masks is None else (masks, masks),
                       None if scales is None else (scales, scales), v)
        assert list(got) == list(ref), f"{name}: keys {list(got)} vs {list(ref)}"
        util.assert_same(got, ref, label=name)
        assert got["qinside"].any(), name


def test_outdoor_832_masks_and_scales_bitwise():
    case = BASELINE_CASES["out4"]
    model, _, _ = util.build_model(case, DEV)
    imgs, masks, scales = util.frames(case)
    bank = model.extract_features(imgs, masks)
    idx0, idx1 = util.idx([0, 1, 2, 7, 3, 3]), util.idx([4, 5, 6, 0, 3, 7])
    pts = _points(idx0, imgs.shape[2:], scales, 4, q=400)
    got = model.match_points_features(bank, idx0, bank, idx1, pts, scale0=scales, scale1=scales)
    ref = _stacked(model, imgs, idx0, imgs, idx1, pts, (masks, masks), (scales, scales))
    assert list(got) == list(ref)
    util.assert_same(got, ref, label="outdoor 832")
    assert got["qvalid"].any()


def test_chain_with_repeated_indices_and_two_banks():
    """A 5-frame chain t -> t+1 plus repeats, in int32 and int64; and pairs across two banks of different sizes."""
    case = CASE["ds_unequal"]
    model, _, _ = util.build_model(case, DEV)
    d = util.device_inputs(case)
    frames = torch.cat([d["image0"], util.device_inputs(case, seed=7)["image0"], util.device_inputs(case, seed=8)[
        "image0"], util.device_inputs(case, seed=9)["image0"], d["image0"].flip(-1)])
    bank = model.extract_features(frames)
    for dt in (torch.int32, torch.int64):
        idx0, idx1 = util.idx([0, 1, 2, 3, 3, 0]).to(dt), util.idx([1, 2, 3, 4, 4, 1]).to(dt)
        pts = _points(idx0.long(), frames.shape[2:], None, 5)
        pts[4] = pts[3]
        got = model.match_points_features(bank, idx0, bank, idx1, pts)
        ref = _stacked(model, frames, idx0.long(), frames, idx1.long(), pts)
        assert list(got) == list(ref)
        util.assert_same(got, ref, label=f"chain {dt}")
        for k in Q_KEYS:   # the repeated pair answers the same queries the same way
            util.assert_same(got[k][4], got[k][3], label=f"chain {dt}: {k} of the repeated pair")
    other = torch.cat([d["image1"], util.device_inputs(case, seed=7)["image1"]])   # 128 x 104
    bank1 = model.extract_features(other)
    idx0, idx1 = util.idx([0, 4, 2]), util.idx([1, 0, 1])
    pts = _points(idx0, frames.shape[2:], None, 6)
    got = model.match_points_features(bank, idx0, bank1, idx1, pts)
    ref = _stacked(model, frames, idx0, other, idx1, pts)
    assert list(got) == list(ref)
    util.assert_same(got, ref, label="two banks")


def test_torch_backbone_follows_the_match_list_rule():
    """cuDNN may pick other algorithms for another batch shape: the answers agree with the stacked call's under the
    match-list rule of DESIGN.md §5 (the same j for at least 99.5% of the answered queries; where j agrees, qconf within
    rtol 1e-3 and qpts1_f within 0.5 px)."""
    case = CASE["ds_thr0"]
    model, _, _ = util.build_model(case, DEV, backbone_impl="torch")
    imgs, _, _ = util.frames(case)
    bank = model.extract_features(imgs)
    idx0, idx1 = util.idx([0, 1, 2, 0]), util.idx([2, 3, 1, 3])
    pts = _points(idx0, imgs.shape[2:], None, 7)
    got = model.match_points_features(bank, idx0, bank, idx1, pts)
    ref = _stacked(model, imgs, idx0, imgs, idx1, pts)
    assert list(got) == list(ref)
    assert all(got[k].dtype == ref[k].dtype for k in Q_KEYS)
    assert torch.equal(got["qinside"], ref["qinside"]) and torch.equal(got["qpts0_f"], ref["qpts0_f"])
    inside = ref["qinside"]
    same = (got["q_j_ids"] == ref["q_j_ids"]) & inside
    frac = same.sum().item() / inside.sum().item()
    assert frac >= 0.995, frac
    assert torch.allclose(got["qconf"][same], ref["qconf"][same], rtol=1e-3, atol=0)
    assert (got["qpts1_f"][same] - ref["qpts1_f"][same]).abs().max().item() <= 0.5
    util.record("bank_points_torch_backbone", {"same_j": frac, "answered": int(inside.sum())})


# ------------------------------------------------------------------------------------------------ 2-4. guided
def test_all_nan_guide_is_the_unguided_call():
    case = CASE["ds_masked_scaled"]
    model, _, _ = util.build_model(case, DEV)
    imgs, masks, scales = util.frames(case)
    bank = model.extract_features(imgs, masks)
    idx0, idx1 = util.idx([0, 1, 2]), util.idx([2, 3, 0])
    pts = _points(idx0, imgs.shape[2:], scales, 8)
    ref = model.match_points_features(bank, idx0, bank, idx1, pts, scale0=scales, scale1=scales)
    for kind in ("homography", "fundamental"):
        got = model.match_points_features(bank, idx0, bank, idx1, pts, scale0=scales, scale1=scales,
                                          guide=util.guide(kind, np.full((3, 3, 3), np.nan), 4.0))
        assert list(got) == list(ref)
        util.assert_same(got, ref, label=f"NaN {kind} guide")


GUIDED = [("ds_thr0", "homography", 20.0), ("ds_thr0", "fundamental", 10.0), ("ot_thr0", "homography", 20.0),
          ("ds_masked_scaled", "homography", 28.0)]


def _guided_setup(name, kind, radius, precision="split"):
    case = CASE[name]
    model, cfg, _ = util.build_model(case, DEV, match_precision=precision)
    imgs, masks, scales = util.frames(case)
    bank = model.extract_features(imgs, masks)
    n = case["n"]
    idx0, idx1 = util.idx(list(range(n)) + [0]), util.idx(list(range(n, 2 * n)) + [n])
    models = np.repeat((util.F_MODEL if kind == "fundamental" else util.H_MODEL)[None], len(idx0), 0)
    models[-1] = np.nan   # the last pair repeats the first, unguided
    return model, cfg, bank, imgs, masks, scales, idx0, idx1, util.guide(kind, models, radius), models


@pytest.mark.parametrize("name, kind, radius", GUIDED, ids=[f"{g[0]}_{g[1]}" for g in GUIDED])
def test_guided_grid_queries_equal_guided_match_features(name, kind, radius):
    model, _, bank, imgs, masks, scales, idx0, idx1, guide, models = _guided_setup(name, kind, radius)
    mf = model.match_features(bank, idx0, bank, idx1, scales, scales, guide=guide)
    q = model.match_points_features(bank, idx0, bank, idx1, util.bank_grid_points(idx0, bank.hw_c, scales),
                                    scale0=scales, scale1=scales, guide=guide)
    b, i = mf["b_ids"], mf["i_ids"]
    assert len(b) > 0 and (b == len(idx0) - 1).any()
    assert q["qinside"][b, i].all() and q["qvalid"][b, i].all()
    assert torch.equal(q["q_i_ids"][b, i], i)
    for qk, fk in (("q_j_ids", "j_ids"), ("qconf", "mconf"), ("qpts0_f", "mkpts0_c"), ("qpts1_c", "mkpts1_c"),
                   ("qpts1_f", "mkpts1_f"), ("qexpec_f", "expec_f")):
        assert torch.equal(q[qk][b, i], mf[fk]), f"{name} {kind}: {qk} differs from the guided {fk}"
    valid = torch.zeros_like(q["qvalid"])
    valid[b, i] = True
    assert torch.equal(q["qvalid"], valid), "qvalid is not the guided match set"
    assert not (q["qvalid"] & ~q["qmutual"]).any() and not (q["qmutual"] & ~q["qinside"]).any()
    # 4. every answered query's cell pair is admissible (the NaN pair admits all)
    s = None if scales is None else scales.cpu().numpy()
    p0 = G.coarse_points(len(idx0), bank.hw_c, 8.0, None if s is None else s[idx0.cpu().numpy()])
    p1 = G.coarse_points(len(idx0), bank.hw_c, 8.0, None if s is None else s[idx1.cpu().numpy()])
    adm, _ = G.admissible(kind, models, radius, p0, p1)
    ans = q["qinside"].cpu().numpy()
    bb, qq = np.nonzero(ans)
    ii, jj = q["q_i_ids"].cpu().numpy()[bb, qq], q["q_j_ids"].cpu().numpy()[bb, qq]
    assert adm[bb, ii, jj].all(), "an answered guided query's cell pair is outside the band"
    assert 0.005 < adm[:-1].mean() < 0.9, adm[:-1].mean()
    util.record(f"bank_points_guided_grid_{name}_{kind}", {"matches": int(len(b)), "answered": int(ans.sum())})


def test_row_without_an_admissible_column_is_not_answered():
    model, _, bank, imgs, masks, scales, idx0, idx1, _, models = _guided_setup("ds_thr0", "homography", 20.0)
    models = models.copy()
    models[1] = [[1, 0, 1e5], [0, 1, 1e5], [0, 0, 1]]   # pair 1: every cell maps far outside image1
    pts = _points(idx0, imgs.shape[2:], None, 10)
    q = model.match_points_features(bank, idx0, bank, idx1, pts, guide=util.guide("homography", models, 20.0))
    assert q["qinside"][0].any() and q["qinside"][2].all()
    assert not q["qinside"][1].any()
    for k in ("qpts0_f", "qpts1_c", "qpts1_f", "qexpec_f"):
        assert torch.isnan(q[k][1]).all(), k
    assert (q["qconf"][1] == 0).all() and (q["q_i_ids"][1] == -1).all() and (q["q_j_ids"][1] == -1).all()
    assert not (q["qmutual"][1] | q["qvalid"][1]).any()


# ------------------------------------------------------------------------------------------------ 5. vs float64
@pytest.mark.parametrize("kind, radius", [("homography", 20.0), ("fundamental", 10.0)])
def test_guided_offgrid_queries_vs_f64(kind, radius):
    model, cfg, bank, imgs, _, _, idx0, idx1, guide, models = _guided_setup("ds_thr0", kind, radius)
    pts = _points(idx0, imgs.shape[2:], None, 11)
    q = model.match_points_features(bank, idx0, bank, idx1, pts, guide=guide)
    sel = q["qinside"].reshape(-1)
    assert sel.float().mean().item() > 0.95   # rows of the band's corners may have no admissible column
    model.expose_coarse_features = True
    fwd = model.match_features(bank, idx0, bank, idx1)   # the coarse transformer outputs of the pair list
    model.expose_coarse_features = False
    x0, x1 = fwd["_feat_c0"], fwd["_feat_c1"]
    nb, nq = pts.shape[:2]
    hw_i, hw_c, hw_f = bank.hw_i, bank.hw_c, bank.hw_f
    stride = hw_f[0] // hw_c[0]
    p0, p1 = G.coarse_points(nb, hw_c, 8.0), G.coarse_points(nb, hw_c, 8.0)
    adm, _ = G.admissible(kind, models, radius, p0, p1)
    conf64 = R.conf_matrix(R.f64(x0, DEV), R.f64(x1, DEV), cfg["match_coarse"], adm=util.to_dev(adm))
    b_ids = torch.arange(nb, device=DEV)[:, None].expand(-1, nq).reshape(-1)[sel]
    i_ids, j_ids = q["q_i_ids"].reshape(-1)[sel], q["q_j_ids"].reshape(-1)[sel]
    rows = conf64[b_ids, i_ids]
    j64 = rows.argmax(1)
    top = rows.topk(2, dim=1).values
    for k in torch.nonzero(j64 != j_ids).flatten().tolist():   # near-ties of the guided row excepted
        gap = ((top[k, 0] - top[k, 1]) / top[k, 0].clamp(min=1e-30)).item()
        assert gap < 1e-2, f"query {k}: j {int(j_ids[k])} vs f64 {int(j64[k])}"
    assert adm[b_ids.cpu().numpy(), i_ids.cpu().numpy(), j_ids.cpu().numpy()].all()
    # the unanswered queries' rows have no admissible column in the predicate either
    rest = ~sel
    if rest.any():
        cb = torch.arange(nb, device=DEV)[:, None].expand(-1, nq).reshape(-1)[rest].cpu().numpy()
        for b, pt in zip(cb, pts.reshape(-1, 2)[rest].cpu().numpy()):
            _, cell, _ = P.query_cells(pt[None], None, hw_i, hw_c, hw_f)
            assert not adm[b, cell[0, 1] * hw_c[1] + cell[0, 0]].any()
    cells, f0s = [], []
    sel_np = sel.view(nb, nq).cpu().numpy()
    for b in range(nb):
        inside, cell, f0 = P.query_cells(pts[b].cpu().numpy(), None, hw_i, hw_c, hw_f)
        assert inside.all()
        cells.append(cell[sel_np[b]])
        f0s.append(f0[sel_np[b]])
    cell, f0 = np.concatenate(cells), np.concatenate(f0s)
    assert (cell[:, 1] * hw_c[1] + cell[:, 0] == i_ids.cpu().numpy()).all()
    f1 = P.image1_centres(cell, f0, j_ids.cpu().numpy(), hw_c[1], stride)
    assert torch.equal(q["qpts0_f"].reshape(-1, 2)[sel].cpu(), torch.tensor(2.0 * f0, dtype=torch.float32))
    assert torch.equal(q["qpts1_c"].reshape(-1, 2)[sel].cpu(), torch.tensor(2.0 * f1, dtype=torch.float32))
    ff0, ff1 = bank.feat_f[idx0], bank.feat_f[idx1]
    pts1_c = q["qpts1_c"].reshape(-1, 2)[sel]
    refs = {dt: P.fine_stage(model, ff0.to(dt), ff1.to(dt), x0.to(dt), x1.to(dt), b_ids, i_ids, j_ids, f0, f1,
                             pts1_c, hw_i, dtype=dt) for dt in (torch.float64, torch.float32)}
    for k, got in (("qexpec_f", q["qexpec_f"].reshape(-1, 3)[sel]), ("qpts1_f", q["qpts1_f"].reshape(-1, 2)[sel])):
        idx = 0 if k == "qexpec_f" else 1
        ref, emu = refs[torch.float64][idx], refs[torch.float32][idx].double()
        ek, eo = (got.double() - ref).abs().max().item(), (emu - ref).abs().max().item()
        scale = ref.abs().max().item()
        util.record(f"bank_points_guided_offgrid_{kind}_{k}", {"err_kernel_vs_f64": ek, "err_fp32_vs_f64": eo,
                                                              "scale": scale, "answered": int(sel.sum())})
        assert ek <= 4 * eo + 1e-6 * scale, f"{k}: kernel error {ek:.3e} vs fp32 emulation {eo:.3e}"


# ------------------------------------------------------------------------------------------------ 6. stale bank
def test_a_bank_of_stale_weights_raises():
    case = CASE["ds_thr0"]
    model, _, _ = util.build_model(case, DEV)
    imgs, _, _ = util.frames(case)
    bank = model.extract_features(imgs)
    idx = util.idx([0, 1])
    pts = _points(idx, imgs.shape[2:], None, 12, q=8)
    model.match_points_features(bank, idx, bank, idx, pts)
    model.load_state_dict(model.state_dict())
    with pytest.raises(RuntimeError, match="match_points_features: `feats0` was extracted with other backbone weights"):
        model.match_points_features(bank, idx, bank, idx, pts)
