"""Pins the float64 references of tests/ref64.py to the reference's own float64 outputs (the `*_f64` keys of the
goldens) and to the full-attention goldens, before ref64 judges any kernel."""
import copy

import numpy as np
import pytest
import torch

import ref64 as R
import util
from cases import CASES, CM_CASES, build_cfg, build_cm_inputs, build_inputs
from edge_cases import EDGE_CASES, build_edge_cfg
from full_cases import FULL_CASES


def _np(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("case", CM_CASES, ids=[c["name"] for c in CM_CASES])
def test_ref64_coarse_matching_matches_reference_f64(case):
    gold = util.load_golden(case["name"])
    mc = build_cfg(case)["match_coarse"]
    inp = build_cm_inputs(case)
    (h0, w0), (h1, w1) = case["hw0c"], case["hw1c"]
    mask0 = mask1 = m0 = m1 = None
    if "mask0" in inp:
        mask0, mask1 = torch.from_numpy(inp["mask0"]), torch.from_numpy(inp["mask1"])
        m0, m1 = mask0.flatten(-2), mask1.flatten(-2)
    conf = R.conf_matrix(R.f64(inp["feat_c0"]), R.f64(inp["feat_c1"]), mc, m0, m1, case.get("bin_score", 1.0))
    out = R.coarse_match(conf, mc, (h0 * 8, w0 * 8), (h0, w0), (h1, w1), mask0, mask1)
    for k in ("b_ids", "i_ids", "j_ids"):
        np.testing.assert_array_equal(_np(out[k]), gold[k + "_f64"], err_msg=k)
    for k in ("mconf", "mkpts0_c", "mkpts1_c"):
        np.testing.assert_allclose(_np(out[k]), gold[k + "_f64"], rtol=1e-9, atol=1e-12, err_msg=k)
    rows, cols = R.top2(conf)
    np.testing.assert_allclose(_np(rows), gold["row_top2_f64"], rtol=1e-9, atol=1e-15)
    np.testing.assert_allclose(_np(cols), gold["col_top2_f64"], rtol=1e-9, atol=1e-15)


def _model_f64_forward(case, cfg):
    """loftr_b200.LoFTR's parameters, a float64 copy of its PyTorch backbone, then ref64.hot_path."""
    import loftr_b200
    import weights as W
    model = loftr_b200.LoFTR(cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    state = W.make_state(shapes, seed=case.get("wseed", 0))
    if "bin_score" in case:
        state["coarse_matching.bin_score"] = np.asarray(case["bin_score"], np.float32)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    inp = build_inputs(case)
    bb = copy.deepcopy(model.backbone).double()
    with torch.no_grad():
        (c0, f0), (c1, f1) = bb(R.f64(inp["image0"])), bb(R.f64(inp["image1"]))
        opt = lambda k: inp.get(k)
        return R.hot_path(model, c0, c1, f0, f1, inp["image0"].shape[2:], opt("mask0"), opt("mask1"), opt("scale0"),
                          opt("scale1"))


def _check_f64_keys(out, gold):
    for k in ("b_ids", "i_ids", "j_ids"):
        np.testing.assert_array_equal(_np(out[k]), gold[k + "_f64"], err_msg=k)
    np.testing.assert_allclose(_np(out["mconf"]), gold["mconf_f64"], rtol=1e-7, atol=1e-12)
    np.testing.assert_allclose(_np(out["mkpts1_f"]), gold["mkpts1_f_f64"], rtol=0, atol=1e-6)
    rows, cols = R.top2(out["conf_matrix"])
    np.testing.assert_allclose(_np(rows), gold["row_top2_f64"], rtol=1e-7, atol=1e-15)
    np.testing.assert_allclose(_np(cols), gold["col_top2_f64"], rtol=1e-7, atol=1e-15)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_ref64_hot_path_matches_reference_f64(case):
    """Float64 backbone + ref64 against the reference run in float64 end to end (linear attention)."""
    _check_f64_keys(_model_f64_forward(case, build_cfg(case)), util.load_golden(case["name"]))


@pytest.mark.parametrize("case", EDGE_CASES, ids=[c["name"] for c in EDGE_CASES])
def test_ref64_edge_configs_match_reference_f64(case):
    """fine_window_size = 3 (9-row windows) end to end in float64."""
    gold = util.load_golden(case["name"])
    out = _model_f64_forward(case, build_edge_cfg(case))
    _check_f64_keys(out, gold)
    assert gold["fine_pre0"].shape[1] == case["fine_window_size"] ** 2


@pytest.mark.parametrize("case", FULL_CASES, ids=[c["name"] for c in FULL_CASES])
def test_ref64_full_attention_matches_reference(case):
    """Full attention: the float64 keys exactly, and the fp32 taps at the tolerance of the fp32 oracle's tests."""
    gold = util.load_golden(case["name"])
    out = _model_f64_forward(case, build_cfg(case))
    _check_f64_keys(out, gold)
    np.testing.assert_allclose(_np(out["feat_c0"])[:, ::7, ::5], gold["feat_c0_s"], rtol=2e-4, atol=2e-4)
    np.testing.assert_allclose(_np(out["feat_c1"])[:, ::7, ::5], gold["feat_c1_s"], rtol=2e-4, atol=2e-4)
    np.testing.assert_allclose(_np(out["expec_f"]), gold["expec_f"], atol=2e-3)


def test_ref64_full_attention_masked_rows_are_zero():
    """Valid rows equal the reference's FullAttention; padded query rows and rows without a valid key are zero."""
    from full_cases import FA_MODULE_CASE, build_fa_module_inputs
    gold = util.load_golden(FA_MODULE_CASE["name"])
    q, k, v, qm, km = build_fa_module_inputs()
    qm_t, km_t = torch.from_numpy(qm), torch.from_numpy(km)
    out = _np(R.full_attention(R.f64(q), R.f64(k), R.f64(v), qm_t, km_t, block=64))
    np.testing.assert_allclose(out[qm], gold["out"][qm], rtol=1e-5, atol=2e-6)   # the golden is fp32
    assert (out[~qm] == 0).all()
    km_t[0] = False
    assert (_np(R.full_attention(R.f64(q), R.f64(k), R.f64(v), qm_t, km_t))[0] == 0).all()
    lin = _np(R.linear_attention(R.f64(q), R.f64(k), R.f64(v), qm_t, km_t))
    assert (lin[0] == 0).all() and (lin[1][~qm[1]] == 0).all()


@pytest.mark.parametrize("W", [3, 5])
def test_ref64_fine_stage_matches_oracle(W):
    """Fine preprocess (any odd W, corner windows, unequal fine maps) and fine matching against the fp32 oracle."""
    from oracle import loftr_oracle as O
    rs = np.random.RandomState(2)
    n, hc, wc, hc1, wc1 = 2, 5, 6, 4, 7
    f0 = rs.standard_normal((n, 16, hc * 4, wc * 4)).astype(np.float32)
    f1 = rs.standard_normal((n, 16, hc1 * 4, wc1 * 4)).astype(np.float32)
    c0 = rs.standard_normal((n, hc * wc, 32)).astype(np.float32)
    c1 = rs.standard_normal((n, hc1 * wc1, 32)).astype(np.float32)
    b = np.array([0, 0, 1, 1, 1])
    i = np.array([0, wc - 1, hc * wc - wc, hc * wc - 1, 7])
    j = np.array([hc1 * wc1 - 1, 0, wc1 - 1, hc1 * wc1 - wc1, 9])
    w = {"down_proj.weight": rs.standard_normal((16, 32)).astype(np.float32),
         "down_proj.bias": rs.standard_normal(16).astype(np.float32),
         "merge_feat.weight": rs.standard_normal((16, 32)).astype(np.float32),
         "merge_feat.bias": rs.standard_normal(16).astype(np.float32)}
    o0, o1 = O.fine_preprocess(f0, f1, c0, c1, b, i, j, wc, wc1, W, 4, w)
    w64 = {k: R.f64(v) for k, v in w.items()}
    g0, g1 = R.fine_preprocess(R.f64(f0), R.f64(f1), R.f64(c0), R.f64(c1), torch.from_numpy(b), torch.from_numpy(i),
                               torch.from_numpy(j), W, 4, w64)
    np.testing.assert_allclose(_np(g0), o0, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(_np(g1), o1, rtol=1e-5, atol=1e-5)
    mk1 = rs.uniform(0, 50, (5, 2)).astype(np.float32)
    sc = rs.uniform(1, 2, (n, 2)).astype(np.float32)
    # scaled down: near-one-hot heatmaps put std at the clamp, where the fp32 oracle's variance is all rounding
    o0, o1, g0, g1 = o0 * 0.05, o1 * 0.05, g0 * 0.05, g1 * 0.05
    of = O.fine_matching(o0, o1, mk1, mk1, b, (hc * 8, wc * 8), (hc * 4, wc * 4), sc)
    e, m = R.fine_matching(g0, g1, mk1, torch.from_numpy(b), (hc * 8, wc * 8), (hc * 4, wc * 4), sc)
    np.testing.assert_allclose(_np(e), of["expec_f"], atol=1e-5)
    np.testing.assert_allclose(_np(m), of["mkpts1_f"], atol=1e-4)
