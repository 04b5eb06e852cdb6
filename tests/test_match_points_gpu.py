"""`LoFTR.match_points` on the GPU (DESIGN.md §17): every forward match comes back bit for bit from a query at its
mkpts0_c, off-grid queries against float64, the edge cases of rule 1, independence of the queries and graph capture."""
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
Q_KEYS = ("qpts0_f", "qpts1_c", "qpts1_f", "qexpec_f", "qconf", "q_i_ids", "q_j_ids", "qmutual", "qvalid", "qinside")


def _match(model, data, pts, valid0=None):
    out = util.inputs(data)
    model.match_points(out, pts, valid0)
    return out


GRID = [
    ("ds_thr0_border2", CASE["ds_thr0"], {}),
    ("ds_thr0_border0", dict(CASE["ds_thr0"], border_rm=0), {}),
    ("out4_masked_scaled", BASELINE_CASES["out4"], {}),
    ("ds_unequal", CASE["ds_unequal"], {}),
    ("ot_thr0", CASE["ot_thr0"], {}),
    ("ot_prefilter", CASE["ot_prefilter"], {}),
    ("full_attention", dict(CASE["ds_thr0"], coarse_attention="full", fine_attention="full"), {}),
    ("fp16", CASE["ds_thr0"], {"backbone_impl": "b200_fp16", "match_precision": "fp16"}),
]


@pytest.mark.parametrize("name, case, opts", GRID, ids=[g[0] for g in GRID])
def test_grid_queries_equal_the_forward_bit_for_bit(name, case, opts):
    model, _, _ = util.build_model(case, DEV, **opts)
    data = util.device_inputs(case)
    fwd = util.eager(model, data)
    q = _match(model, data, util.grid_points(data))
    n, L = q["qvalid"].shape
    b, i = fwd["b_ids"], fwd["i_ids"]
    if name == "ot_prefilter":   # the prefilter removes every row and column of this pair: nothing is kept or valid
        assert len(b) == 0 and not q["qvalid"].any()
        return
    assert len(b) > 0, name
    assert q["qinside"][b, i].all() and q["qvalid"][b, i].all(), name
    assert torch.equal(q["q_i_ids"][b, i], i), name
    for qk, fk in (("q_j_ids", "j_ids"), ("qconf", "mconf"), ("qpts0_f", "mkpts0_c"), ("qpts1_c", "mkpts1_c"),
                   ("qpts1_f", "mkpts1_f"), ("qexpec_f", "expec_f")):
        assert torch.equal(q[qk][b, i], fwd[fk]), f"{name}: {qk} differs from the forward's {fk}"
    others = torch.ones(n, L, dtype=torch.bool, device=DEV)
    others[b, i] = False
    assert not q["qvalid"][others].any(), f"{name}: a cell the forward drops has qvalid"
    # qvalid implies mutual and inside; masked cells are not inside
    assert not (q["qvalid"] & ~q["qmutual"]).any() and not (q["qmutual"] & ~q["qinside"]).any()
    if "mask0" in data:
        assert not q["qinside"][~data["mask0"].reshape(n, L)].any()


# ------------------------------------------------------------------------------------------------ off-grid vs f64
def _offgrid_points(n, h, w, seed):
    """Sub-pixel points, image corners and edges (windows partly outside on both sides), and the last cell row and
    column -> [n, Q, 2]."""
    rs = np.random.RandomState(seed)
    edges = [(0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1), (0.4, 37.3), (w - 1.2, 21.7), (55.5, 0.3),
             (61.1, h - 1.4), (w - 4.6, h - 4.6), (w - 9.0, h - 9.0), (3.9, 4.1), (w / 2 + 0.49, h / 2 + 1.51)]
    pts = []
    for _ in range(n):
        sub = np.stack([rs.uniform(0, w - 1, 150), rs.uniform(0, h - 1, 150)], 1)
        pts.append(np.concatenate([np.asarray(edges, np.float64), sub], 0))
    return torch.tensor(np.stack(pts), dtype=torch.float32, device=DEV)


@pytest.mark.parametrize("case", [CASE["ds_thr0"], CASE["ds_unequal"]], ids=["ds_thr0", "ds_unequal"])
def test_offgrid_queries_vs_f64(case):
    model, cfg, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    n, _, h, w = data["image0"].shape
    pts = _offgrid_points(n, h, w, 5)
    q = _match(model, data, pts)
    assert q["qinside"].all()
    # the kernel's own stage inputs: backbone fine maps and coarse transformer outputs
    model.expose_coarse_features = True
    fwd = util.eager(model, data)
    model.expose_coarse_features = False
    with torch.no_grad():
        if data["image0"].shape == data["image1"].shape:
            _, ff = model._backbone(torch.cat([data["image0"], data["image1"]]))
            ff0, ff1 = ff[:n], ff[n:]
        else:
            (_, ff0), (_, ff1) = model._backbone(data["image0"]), model._backbone(data["image1"])
    x0, x1 = fwd["_feat_c0"], fwd["_feat_c1"]
    hw_i, hw_c, hw_f = fwd["hw0_i"], fwd["hw0_c"], fwd["hw0_f"]
    (h1c, w1c), stride = fwd["hw1_c"], hw_f[0] // hw_c[0]
    # j against the float64 row arg-max, near-ties excepted
    conf64 = R.conf_matrix(R.f64(x0, DEV), R.f64(x1, DEV), cfg["match_coarse"])
    b_ids = torch.arange(n, device=DEV)[:, None].expand(-1, pts.shape[1]).reshape(-1)
    i_ids, j_ids = q["q_i_ids"].reshape(-1), q["q_j_ids"].reshape(-1)
    j64 = conf64[b_ids, i_ids].argmax(1)
    for k in torch.nonzero(j64 != j_ids).flatten().tolist():
        b = int(b_ids[k])
        r, _ = util.near_tie_top2_f64(x0[b].cpu().numpy(), x1[b].cpu().numpy(), cfg["match_coarse"])
        r = r[int(i_ids[k])]
        assert abs(r[0] - r[1]) / max(r[0], 1e-30) < 1e-2, f"query {k}: j {int(j_ids[k])} vs f64 {int(j64[k])}"
    # rules 1, 2 and 4 from the numpy statement, then the fine stage from the kernel's own j
    cells, f0s = [], []
    for b in range(n):
        inside, cell, f0 = P.query_cells(pts[b].cpu().numpy(), None, hw_i, hw_c, hw_f)
        assert inside.all()
        cells.append(cell)
        f0s.append(f0)
    cell, f0 = np.concatenate(cells), np.concatenate(f0s)
    assert (cell[:, 1] * hw_c[1] + cell[:, 0] == i_ids.cpu().numpy()).all()
    f1 = P.image1_centres(cell, f0, j_ids.cpu().numpy(), w1c, stride)
    assert torch.equal(q["qpts0_f"].reshape(-1, 2).cpu(), torch.tensor(2.0 * f0, dtype=torch.float32))
    assert torch.equal(q["qpts1_c"].reshape(-1, 2).cpu(), torch.tensor(2.0 * f1, dtype=torch.float32))
    pts1_c = q["qpts1_c"].reshape(-1, 2)
    refs = {}
    for dt in (torch.float64, torch.float32):
        refs[dt] = P.fine_stage(model, ff0.to(dt), ff1.to(dt), x0.to(dt), x1.to(dt), b_ids, i_ids, j_ids, f0, f1,
                                pts1_c, hw_i, dtype=dt)
    for k, got in (("qexpec_f", q["qexpec_f"].reshape(-1, 3)), ("qpts1_f", q["qpts1_f"].reshape(-1, 2))):
        idx = 0 if k == "qexpec_f" else 1
        ref, emu = refs[torch.float64][idx], refs[torch.float32][idx].double()
        ek, eo = (got.double() - ref).abs().max().item(), (emu - ref).abs().max().item()
        scale = ref.abs().max().item()
        util.record(f"points_offgrid_{case['name']}_{k}", {"err_kernel_vs_f64": ek, "err_fp32_vs_f64": eo,
                                                           "scale": scale})
        assert ek <= 4 * eo + 1e-6 * scale, f"{k}: kernel error {ek:.3e} vs fp32 emulation {eo:.3e}"


# ------------------------------------------------------------------------------------------------ edges
def _assert_unanswered(q, sel, label):
    for k in ("qpts0_f", "qpts1_c", "qpts1_f", "qexpec_f"):
        assert torch.isnan(q[k][sel]).all(), (label, k)
    assert (q["qconf"][sel] == 0).all() and (q["q_i_ids"][sel] == -1).all() and (q["q_j_ids"][sel] == -1).all()
    for k in ("qmutual", "qvalid", "qinside"):
        assert not q[k][sel].any(), (label, k)


def test_edges_valid0_nan_outside_masked_and_duplicates():
    case = CASE["ot_masked"]   # n = 1, 128 x 128, image0 valid in 128 x 96: cells with x >= 12 are masked
    model, _, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    s = data["scale0"][0]
    img = lambda x, y: [x * float(s[0]), y * float(s[1])]   # network pixels -> source pixels
    nan = float("nan")
    pts = [img(20.3, 30.7), img(20.3, 30.7),   # duplicates
           img(20.3, 30.7),                    # valid0 false
           [nan, 5.0], [5.0, float("inf")],    # not finite
           img(-0.5, 3.0), img(3.0, 127.5),    # outside [0, W0 - 1] x [0, H0 - 1]
           img(110.0, 40.0),                   # a masked cell (x >= 96)
           img(91.0, 126.9)]                   # the last unmasked cell column (91 / 8 + 0.5 -> 11), last row
    pts = torch.tensor([pts], dtype=torch.float32, device=DEV)
    valid0 = torch.ones(1, pts.shape[1], dtype=torch.bool, device=DEV)
    valid0[0, 2] = False
    q = _match(model, data, pts, valid0)
    inside = q["qinside"][0].tolist()
    assert inside == [True, True, False, False, False, False, False, False, True]
    _assert_unanswered(q, ~q["qinside"], "edges")
    for k in Q_KEYS:
        assert torch.equal(q[k][0, 0], q[k][0, 1]), k
    assert q["q_i_ids"][0, 8].item() == 15 * 16 + 11


def test_row_without_a_valid_column_has_no_answer():
    case = CASE["ds_masked_scaled"]
    model, _, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    data["mask1"][1] = False   # pair 1: every column masked
    pts = torch.tensor([[[40.0, 40.0], [64.0, 32.0]]] * 2, dtype=torch.float32, device=DEV) * data["scale0"][:, None]
    q = _match(model, data, pts)
    assert q["qinside"][0].all()
    _assert_unanswered(q, (slice(1, 2),), "masked pair")


def test_q1_n1_and_q0():
    case = CASE["ds_unequal"]
    model, _, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    q = _match(model, data, torch.tensor([[[17.25, 33.5]]], device=DEV))
    assert q["qinside"].shape == (1, 1) and q["qinside"].item()
    assert q["qpts1_f"].shape == (1, 1, 2) and q["qexpec_f"].shape == (1, 1, 3)
    launches = _lib.load().lb_launch_count
    n_launch = launches()
    e = _match(model, data, torch.empty(1, 0, 2, device=DEV))
    assert launches() == n_launch   # Q = 0 launches nothing
    for k in Q_KEYS:
        assert e[k].shape[:2] == (1, 0) and e[k].dtype == q[k].dtype, k


# ------------------------------------------------------------------------------------------------ independence
def test_queries_are_independent():
    case = CASE["ds_thr0"]
    model, _, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    n, _, h, w = data["image0"].shape
    pts = _offgrid_points(n, h, w, 9)
    full = _match(model, data, pts)
    again = _match(model, data, pts)
    util.assert_same(again, full, Q_KEYS, "two eager calls")
    for sub in (torch.arange(0, pts.shape[1], 7), torch.tensor([5]), torch.arange(pts.shape[1] - 3, pts.shape[1])):
        part = _match(model, data, pts[:, sub.to(DEV)].contiguous())
        for k in Q_KEYS:
            assert torch.equal(part[k], full[k][:, sub.to(DEV)]), k


# ------------------------------------------------------------------------------------------------ graph capture
def test_graph_capture_replays_new_points():
    case = CASE["ds_masked_scaled"]
    model, _, _ = util.build_model(case, DEV)
    data = util.device_inputs(case)
    n, _, h, w = data["image0"].shape
    s = data["scale0"][:, None]
    pts_a = (_offgrid_points(n, h, w, 1) * s).contiguous()
    pts_b = (_offgrid_points(n, h, w, 2) * s).contiguous()
    static_in, static_pts = util.inputs(data), pts_a.clone()
    model.match_points(dict(static_in), static_pts)   # eager warm-up (weight packing)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        model.match_points(dict(static_in), static_pts)
    torch.cuda.current_stream().wait_stream(side)
    graph, out = torch.cuda.CUDAGraph(), dict(static_in)
    with torch.cuda.graph(graph):
        model.match_points(out, static_pts)
    for pts in (pts_b, pts_a):
        static_pts.copy_(pts)
        graph.replay()
        torch.cuda.synchronize()
        util.assert_same(out, _match(model, data, pts), Q_KEYS, "graph replay")
