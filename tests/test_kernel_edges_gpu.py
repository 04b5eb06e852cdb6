"""Every matching kernel against the float64 references of tests/ref64.py, at the tile, chunk, split and mask
boundaries where its branches change.  Each grid point names the branch it covers; where the branch depends on derived
launch parameters, the test recomputes them (from the SM count of the device) and asserts that the case still hits
them.

Tolerances:
- match lists: `util.compare_matches` (overlap >= 99.5 %, mconf rtol 1e-3, keypoints < 0.5 px), ref64 as the reference
  and, through its top-2 statistics, as the adjudicator of every non-shared match;
- dense outputs: the kernel's largest error against float64 is at most 4x that of the fp32 numpy oracle on the same
  input, plus 1e-6 (the kernels claim fp32-class accuracy, DESIGN.md §2).
Every test records its largest errors through `util.record`."""
import numpy as np
import pytest
import torch

import ref64 as R
import util
import weights as WT
from cases import CASES, BASELINE_CASES, build_cfg, build_cm_inputs, build_inputs
from edge_cases import EDGE_CASES, build_edge_cfg
from oracle import loftr_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# launch constants mirrored from csrc/engine.cu and csrc/gemm_split.cuh
BLOCK_M, SCORE_BN, MAX_CHUNKS, KV_SPLITS = 128, 256, 32, 8


def _t(x, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(x)).to(DEV)
    return t if dtype is None else t.to(dtype)


def _np(t):
    return t.detach().cpu().numpy()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


# Grid points where the kernel's error exceeds 4x the fp32 oracle's (measured on an H100 SXM, 132 SMs).  The bound is
# kept; these points xfail with the reason below after passing a coarse sanity bound (1e-5 of the output scale).
# Products are exact to 2^-22 (fp16 hi + lo planes, DESIGN.md §2), 4x fp32's unit roundoff, so a ratio near 4 is the
# design's own floor.  Full attention splits the softmax weights P (all <= 1, mostly far below 2^-3) into planes in
# registers; their fp16 `lo` plane is then subnormal, so P carries an absolute 2^-25 rather than a relative 2^-22 error.
# With one token (L = S = 1) the oracle sums a single term and its own error is unusually small.
RATIO_FINDINGS = {
    "tf_coarse_linear_n1_L1_S1": "one token: the fp32 oracle's error is a single rounding, the kernel's is 2^-22",
    "tf_coarse_full_n1_L1_S1": "one token: the fp32 oracle's error is a single rounding, the kernel's is 2^-22",
    "tf_coarse_full_n1_L4800_S300": "full attention: subnormal fp16 lo plane of the softmax weights P",
    "tf_coarse_full_n1_L300_S4800": "full attention: subnormal fp16 lo plane of the softmax weights P",
    "tf_coarse_full_2_70_1_None": "full attention, one key: P = 1 exactly, the oracle's error is unusually small",
    "tf_coarse_full_2_70_64_None": "full attention: subnormal fp16 lo plane of the softmax weights P",
}


def _bound(name, got, ref, oracle, extra=None, finding=None):
    """Dense-output rule: max|kernel - fp64| <= 4 * max|fp32 oracle - fp64| + 1e-6."""
    got, ref, oracle = (np.asarray(_np(x) if torch.is_tensor(x) else x, np.float64) for x in (got, ref, oracle))
    assert got.shape == ref.shape == oracle.shape, (got.shape, ref.shape, oracle.shape)
    ek = float(np.abs(got - ref).max()) if got.size else 0.0
    eo = float(np.abs(oracle - ref).max()) if got.size else 0.0
    util.record(name, {"err_kernel_vs_f64": ek, "err_fp32_oracle_vs_f64": eo, "ratio": ek / max(eo, 1e-30),
                       "scale": float(np.abs(ref).max()) if ref.size else 0.0, **(extra or {})})
    if finding is not None and ek > 4 * eo + 1e-6:
        assert ek <= 1e-5 * float(np.abs(ref).max()), f"{name}: kernel error {ek:.3e} (fp32 oracle {eo:.3e})"
        pytest.xfail(f"{name}: ratio {ek / max(eo, 1e-30):.2f} > 4: {finding}")
    assert ek <= 4 * eo + 1e-6, f"{name}: kernel error {ek:.3e} vs fp32 oracle {eo:.3e}"
    return ek, eo


def _model(W=5, coarse="linear", fine="linear", device=DEV):
    """loftr_b200.LoFTR with the deterministic weights of tests/golden/weights.py and the given window / attentions."""
    import loftr_b200
    cfg = build_cfg(CASES[0])
    cfg["fine_window_size"] = W
    cfg["coarse"]["attention"], cfg["fine"]["attention"] = coarse, fine
    model = loftr_b200.LoFTR(cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    state = WT.make_state(shapes, seed=0)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    return model.to(device), cfg, state


# ------------------------------------------------------------------------------------------------ coarse matching
def cm_launch(n, L, S, sms):
    """Mirror of lb_coarse_match's chunking (engine.cu pick_chunks, kMaxChunks, the tpc / n_chunks mirror)."""
    m_tiles, n_tiles = _cdiv(L, BLOCK_M), _cdiv(S, SCORE_BN)
    raw = 1
    while n * m_tiles * raw < 40 * sms and raw < n_tiles:
        raw += 1
    chunks = min(raw, MAX_CHUNKS)
    tpc = _cdiv(n_tiles, chunks)
    n_chunks = _cdiv(n_tiles, tpc)
    return {"raw": raw, "chunks": chunks, "tpc": tpc, "n_chunks": n_chunks, "n_tiles": n_tiles, "m_tiles": m_tiles,
            "partial_last_chunk": n_tiles % tpc != 0, "partial_last_col_block": S % 32 != 0}


def _cp(cid, **kw):
    return pytest.param(kw, id=cid)


_GRID = {127: (1, 127), 128: (8, 16), 129: (3, 43), 255: (15, 17), 256: (16, 16), 257: (1, 257)}
CM_SHAPES = [_cp(f"L{L}_S{S}", n=3, hw0c=_GRID[L], hw1c=_GRID[S], border_rm=0)
             for L in (127, 128, 129) for S in (255, 256, 257)] + [
    _cp("grid_1x1", n=2, hw0c=(1, 1), hw1c=(1, 1), border_rm=0),
    _cp("n6_48_tokens", n=6, hw0c=(6, 8), hw1c=(8, 6), border_rm=0),
    # S = 18915: 74 column tiles -> the chunk count is clamped to 32 (tpc 3, last chunk 2 tiles) and the last 32-column
    # block holds 3 columns, so the shared-reference fast path of the LSE epilogue (epilogues.cuh:1132) is skipped there
    _cp("L128_S18915_chunk_clamp", n=1, hw0c=(8, 16), hw1c=(97, 195), border_rm=2,
        expect={"clamped": True, "partial_last_chunk": True, "partial_last_col_block": True}),
    _cp("L18915_S128_one_col_tile", n=1, hw0c=(97, 195), hw1c=(8, 16), border_rm=2, expect={"n_chunks": 1}),
    # pair 0 fully valid (image 1 padded at the bottom), pair 1 three valid columns (< 2*border_rm + 1: every match
    # removed), pair 2 one valid column
    _cp("masks_narrow", n=3, hw0c=(12, 16), hw1c=(12, 16), border_rm=2,
        valid0c=[(12, 16), (12, 3), (12, 1)], valid1c=[(10, 16), (9, 16), (12, 16)], no_match_pairs=(1, 2)),
]
OT_PARAMS = [_cp(f"iters{it}_{'pre' if pre else 'nopre'}_bin{b:g}", n=2, hw0c=(10, 14), hw1c=(12, 12), border_rm=2,
                 skh_iters=it, prefilter=pre, bin_score=b)
             for it in (0, 1, 3, 10) for pre in (False, True) for b in (-3.0, 1.0, 6.0)]
DS_PARAMS = [_cp(f"temp{t:g}", n=2, hw0c=(10, 14), hw1c=(12, 12), border_rm=2, temperature=t) for t in (0.05, 0.2)] + [
    _cp("border4", n=2, hw0c=(12, 16), hw1c=(14, 14), border_rm=4)]


def _run_cm(case, match_type, name, return_conf=False):
    n, (h0, w0), (h1, w1) = case["n"], case["hw0c"], case["hw1c"]
    L, S = h0 * w0, h1 * w1
    lp = cm_launch(n, L, S, _sms())
    exp = case.get("expect", {})
    if exp.get("clamped"):
        assert lp["raw"] > MAX_CHUNKS and lp["chunks"] == MAX_CHUNKS, lp
    for k in ("partial_last_chunk", "partial_last_col_block", "n_chunks"):
        if k in exp:
            assert lp[k] == exp[k], (k, lp)
    ot = match_type == "sinkhorn"
    cm_case = {"n": n, "hw0c": case["hw0c"], "hw1c": case["hw1c"], "amp": 3.0 if ot else 1.6, "frac": 0.6,
               "iseed": 17}
    if "valid0c" in case:
        cm_case.update(valid0c=case["valid0c"], valid1c=case["valid1c"])
    inp = build_cm_inputs(cm_case)
    mc = build_cfg({"thr": case.get("thr", 0.0), "match_type": match_type, "prefilter": case.get("prefilter", False),
                    "border_rm": case["border_rm"]})["match_coarse"]
    mc["skh_iters"] = case.get("skh_iters", 3)
    mc["dsmax_temperature"] = case.get("temperature", 0.1)
    mc["return_conf_matrix"] = return_conf
    bin_score = case.get("bin_score", 1.0)
    import loftr_b200.loftr as LM
    mod = LM.CoarseMatching(mc).eval().to(DEV)
    if ot:
        mod.bin_score.data = torch.tensor(bin_score, device=DEV)
    data = {"hw0_i": (h0 * 8, w0 * 8), "hw1_i": (h1 * 8, w1 * 8), "hw0_c": (h0, w0), "hw1_c": (h1, w1)}
    mask0 = mask1 = m0 = m1 = None
    if "mask0" in inp:
        data["mask0"], data["mask1"] = mask0, mask1 = _t(inp["mask0"]), _t(inp["mask1"])
        m0, m1 = mask0.flatten(-2), mask1.flatten(-2)
    mod(_t(inp["feat_c0"]), _t(inp["feat_c1"]), data, m0, m1)
    got = {k: _np(data[k]) for k in ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c")}
    conf = R.conf_matrix(R.f64(inp["feat_c0"], DEV), R.f64(inp["feat_c1"], DEV), mc, m0, m1, bin_score)
    ref = R.coarse_match(conf, mc, data["hw0_i"], (h0, w0), (h1, w1), mask0, mask1)
    ref = {k: _np(v) for k, v in ref.items()}
    rows, cols = R.top2(conf)
    gold = {"row_top2_f64": _np(rows), "col_top2_f64": _np(cols)}
    stats = util.compare_matches(got, ref, gold, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995, label=name)
    for p in case.get("no_match_pairs", ()):
        assert not (got["b_ids"] == p).any() and not (ref["b_ids"] == p).any(), f"{name}: pair {p} has matches"
    util.record(name, {**stats, **{k: v for k, v in lp.items() if not isinstance(v, bool)}})
    return data, conf, inp, mc, stats


@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
@pytest.mark.parametrize("case", CM_SHAPES)
def test_coarse_matching_shapes_vs_f64(case, match_type):
    _, _, _, _, stats = _run_cm(case, match_type, f"cm_{match_type}")
    assert stats["n"] > 0 or case["hw0c"] == (1, 1) or match_type == "sinkhorn"


@pytest.mark.parametrize("case", OT_PARAMS)
def test_sinkhorn_parameters_vs_f64(case):
    _run_cm(case, "sinkhorn", "cm_sinkhorn_params")


@pytest.mark.parametrize("case", DS_PARAMS)
def test_dual_softmax_parameters_vs_f64(case):
    _, _, _, _, stats = _run_cm(case, "dual_softmax", "cm_dual_softmax_params")
    assert stats["n"] > 0


@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
def test_conf_matrix_multi_chunk_vs_f64(match_type):
    """return_conf_matrix at a shape with several column chunks, elementwise against float64."""
    case = {"n": 2, "hw0c": (12, 20), "hw1c": (40, 60), "border_rm": 2}
    lp = cm_launch(2, 240, 2400, _sms())
    assert lp["n_chunks"] > 1, lp
    data, conf, inp, mc, _ = _run_cm(case, match_type, f"cm_conf_matrix_{match_type}", return_conf=True)
    got, ref = _np(data["conf_matrix"]).astype(np.float64), _np(conf)
    rel = np.abs(got - ref) / np.maximum(ref, 1e-30)
    big = ref > 1e-30
    util.record(f"cm_conf_matrix_{match_type}", {"rel_max": float(rel[big].max()), "abs_max": float(np.abs(got - ref).max())})
    np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-12)


# ------------------------------------------------------------------------------------------------ transformers
def kv_splits(n_groups, rows, sms):
    """Mirror of the split-K count of kv_gemm_kernel (engine.cu tf_linear_attention_coarse)."""
    kb_total = _cdiv(rows, 64)
    parts_cap = max(_cdiv(rows, BLOCK_M), KV_SPLITS)
    s = min(max(sms // (2 * n_groups), 1), kb_total, parts_cap)
    return _cdiv(kb_total, _cdiv(kb_total, s))


def _tf_check(name, tf, attention, f0, f1, m0=None, m1=None):
    import full_oracle as FO
    lw = R.layer_weights(tf, DEV)
    names, nhead = tf.layer_names, tf.nhead
    t = lambda m: None if m is None else _t(m)
    g0, g1 = tf(_t(f0), _t(f1), t(m0), t(m1))
    r0, r1 = R.transformer(R.f64(f0, DEV), R.f64(f1, DEV), lw, names, nhead, t(m0), t(m1), attention)
    ow = [{k: _np(v).astype(np.float32) for k, v in w.items()} for w in lw]
    o0, o1 = FO.local_feature_transformer(f0, f1, ow, names, nhead, m0, m1, attention)
    finding = RATIO_FINDINGS.get(name)
    errs = [_bound(name + "_feat0", g0, r0, o0, finding=finding), _bound(name + "_feat1", g1, r1, o1, finding=finding)]
    return errs


def _feats(n, L, S, c, seed):
    rs = np.random.RandomState(seed)
    f0 = rs.standard_normal((n, L, c)).astype(np.float32)
    f1 = rs.standard_normal((n, S, c)).astype(np.float32)
    return f0, f1


COARSE_TF = [_cp(f"n{n}_L{L}_S{S}", n=n, L=L, S=S)
             for n, L, S in ((1, 1, 1), (3, 65, 63), (3, 127, 129), (1, 4800, 300), (1, 300, 4800))]
FULL_ONLY = [_cp(f"S{S}", n=2, L=70, S=S) for S in (1, 63, 64, 65)] + [
    _cp("keys_0_64_masked", n=2, L=90, S=150, key_hole=(0, 64)),
    _cp("keys_64_128_masked", n=2, L=90, S=200, key_hole=(64, 128))]


@pytest.mark.parametrize("attention", ["linear", "full"])
@pytest.mark.parametrize("case", COARSE_TF)
def test_coarse_transformer_shapes_vs_f64(case, attention):
    model, _, _ = _model(coarse=attention)
    f0, f1 = _feats(case["n"], case["L"], case["S"], 256, 31)
    _tf_check(f"tf_coarse_{attention}_n{case['n']}_L{case['L']}_S{case['S']}", model.loftr_coarse, attention, f0, f1)


@pytest.mark.parametrize("case", FULL_ONLY)
def test_full_attention_key_tiles_vs_f64(case):
    """S below, at and just past one 64-key tile; a fully masked first / middle key tile (the -inf key bias)."""
    model, _, _ = _model(coarse="full")
    n, L, S = case["n"], case["L"], case["S"]
    f0, f1 = _feats(n, L, S, 256, 37)
    m0 = m1 = None
    if "key_hole" in case:
        m0, m1 = np.ones((n, L), bool), np.ones((n, S), bool)
        m1[:, case["key_hole"][0]:case["key_hole"][1]] = False
    _tf_check(f"tf_coarse_full_{'_'.join(map(str, (n, L, S)))}_{case.get('key_hole')}", model.loftr_coarse, "full",
              f0, f1, m0, m1)


@pytest.mark.parametrize("attention", ["linear", "full"])
def test_coarse_transformer_split_k_vs_f64(attention):
    """The same 200 x 200 data at n = 2 (split-K K^T V) and n = 67 (splits = 1): both within the fp64 bound."""
    sms = _sms()
    assert kv_splits(2, 200, sms) > 1 and kv_splits(67, 200, sms) == 1
    model, _, _ = _model(coarse=attention)
    f0, f1 = _feats(2, 200, 200, 256, 41)
    _tf_check(f"tf_coarse_{attention}_n2_200", model.loftr_coarse, attention, f0, f1)
    reps = _cdiv(67, 2)
    f0b, f1b = np.tile(f0, (reps, 1, 1))[:67], np.tile(f1, (reps, 1, 1))[:67]
    _tf_check(f"tf_coarse_{attention}_n67_200_splits1", model.loftr_coarse, attention, f0b, f1b)


@pytest.mark.parametrize("attention", ["linear", "full"])
def test_coarse_transformer_fully_masked_images_vs_f64(attention):
    """Pair 1: every key of image 1 masked; pair 2: every query of image 0 masked; pair 0: random padding."""
    model, _, _ = _model(coarse=attention)
    n, L, S = 3, 130, 97
    f0, f1 = _feats(n, L, S, 256, 43)
    rs = np.random.RandomState(44)
    m0, m1 = rs.uniform(size=(n, L)) > 0.2, rs.uniform(size=(n, S)) > 0.3
    m1[1] = False
    m0[2] = False
    _tf_check(f"tf_coarse_{attention}_fully_masked", model.loftr_coarse, attention, f0, f1, m0, m1)


WINDOWS = [_cp("W3_9rows", n=37, l=9, s=9), _cp("W5_25rows", n=37, l=25, s=25),
           _cp("unequal_25_vs_9", n=37, l=25, s=9), _cp("one_window", n=1, l=25, s=25),
           _cp("5003_windows", n=5003, l=9, s=9)]


@pytest.mark.parametrize("attention", ["linear", "full"])
@pytest.mark.parametrize("case", WINDOWS)
def test_window_transformer_vs_f64(case, attention):
    model, _, _ = _model(fine=attention)
    f0, f1 = _feats(case["n"], case["l"], case["s"], 128, 47)
    if attention == "full" and case["l"] != case["s"]:
        with pytest.raises(RuntimeError, match="equal window sizes"):   # built for equal windows only
            model.loftr_fine(_t(f0), _t(f1))
        return
    _tf_check(f"tf_fine_{attention}_n{case['n']}_{case['l']}x{case['s']}", model.loftr_fine, attention, f0, f1)


# ------------------------------------------------------------------------------------------------ fine level
@pytest.mark.parametrize("layout", ["nchw", "nhwc", "channel_slice"])
@pytest.mark.parametrize("W", [3, 5])
def test_fine_preprocess_vs_f64(W, layout):
    """Windows at all four corners of both grids, unequal fine maps, three memory layouts of the fine features."""
    model, _, state = _model(W=W)
    rs = np.random.RandomState(51)
    n, (hc0, wc0), (hc1, wc1) = 2, (9, 12), (11, 7)
    f0 = rs.standard_normal((n, 128, hc0 * 4, wc0 * 4)).astype(np.float32)
    f1 = rs.standard_normal((n, 128, hc1 * 4, wc1 * 4)).astype(np.float32)
    c0 = rs.standard_normal((n, hc0 * wc0, 256)).astype(np.float32)
    c1 = rs.standard_normal((n, hc1 * wc1, 256)).astype(np.float32)
    corners0 = [0, wc0 - 1, (hc0 - 1) * wc0, hc0 * wc0 - 1]
    corners1 = [0, wc1 - 1, (hc1 - 1) * wc1, hc1 * wc1 - 1]
    b = np.array([0] * 4 + [1] * 4 + [0, 1] * 20, np.int64)
    i = np.array(corners0 + corners0[::-1] + list(rs.randint(0, hc0 * wc0, 40)), np.int64)
    j = np.array(corners1 + corners1[1:] + corners1[:1] + list(rs.randint(0, hc1 * wc1, 40)), np.int64)
    order = np.argsort(b, kind="stable")
    b, i, j = b[order], i[order], j[order]
    tf0, tf1 = _t(f0), _t(f1)
    if layout == "nhwc":
        tf0, tf1 = tf0.contiguous(memory_format=torch.channels_last), tf1.contiguous(memory_format=torch.channels_last)
    elif layout == "channel_slice":
        big0 = torch.randn(n, 300, hc0 * 4, wc0 * 4, device=DEV)
        big1 = torch.randn(n, 300, hc1 * 4, wc1 * 4, device=DEV)
        big0[:, 100:228], big1[:, 100:228] = tf0, tf1
        tf0, tf1 = big0[:, 100:228], big1[:, 100:228]
        assert not tf0.is_contiguous()
    data = {"hw0_i": (hc0 * 8, wc0 * 8), "hw0_c": (hc0, wc0), "hw1_c": (hc1, wc1), "hw0_f": tuple(f0.shape[2:]),
            "hw1_f": tuple(f1.shape[2:]), "b_ids": _t(b), "i_ids": _t(i), "j_ids": _t(j)}
    g0, g1 = model.fine_preprocess(tf0, tf1, _t(c0), _t(c1), data)
    fw = {k: state[f"fine_preprocess.{k}"] for k in ("down_proj.weight", "down_proj.bias", "merge_feat.weight",
                                                      "merge_feat.bias")}
    o0, o1 = O.fine_preprocess(f0, f1, c0, c1, b, i, j, wc0, wc1, W, 4, fw)
    r0, r1 = R.fine_preprocess(R.f64(f0, DEV), R.f64(f1, DEV), R.f64(c0, DEV), R.f64(c1, DEV), _t(b), _t(i), _t(j), W,
                               4, {k: R.f64(v, DEV) for k, v in fw.items()})
    _bound(f"fine_pre_W{W}_{layout}_0", g0, r0, o0)
    _bound(f"fine_pre_W{W}_{layout}_1", g1, r1, o1)


def _fine_match(W, f0, f1, seed=0, name="fine_match"):
    m = f0.shape[0]
    rs = np.random.RandomState(seed)
    mk1 = rs.uniform(0, 100, (m, 2)).astype(np.float32)
    b = np.zeros(m, np.int64)
    scale1 = np.array([[1.5, 1.25]], np.float32)
    hw0_i, hw0_f = (96, 128), (48, 64)
    data = {"hw0_i": hw0_i, "hw0_f": hw0_f, "b_ids": _t(b), "mkpts0_c": _t(mk1), "mkpts1_c": _t(mk1),
            "scale0": _t(scale1), "scale1": _t(scale1), "mconf": torch.ones(m, device=DEV)}
    from loftr_b200.loftr import FineMatching
    FineMatching()(_t(f0), _t(f1), data)
    of = O.fine_matching(f0, f1, mk1, mk1, b, hw0_i, hw0_f, scale1)
    re, rk = R.fine_matching(R.f64(f0, DEV), R.f64(f1, DEV), mk1, _t(b), hw0_i, hw0_f, scale1)
    _bound(name + "_expec_f", data["expec_f"], re, of["expec_f"])
    _bound(name + "_mkpts1_f", data["mkpts1_f"], rk, of["mkpts1_f"])
    return _np(data["expec_f"]), _np(re)


@pytest.mark.parametrize("M", [1, 40000])
@pytest.mark.parametrize("W", [3, 5])
def test_fine_matching_random_vs_f64(W, M):
    rs = np.random.RandomState(61)
    f0 = rs.standard_normal((M, W * W, 128)).astype(np.float32)
    f1 = rs.standard_normal((M, W * W, 128)).astype(np.float32)
    _fine_match(W, f0, f1, 1, f"fine_match_W{W}_M{M}")


@pytest.mark.parametrize("W", [3, 5])
def test_fine_matching_near_one_hot_and_flat(W):
    """One cell holding > 1 - 1e-6 of the mass (at a corner: expec_f on +-1, std at the 1e-10 clamp), and exactly flat
    heatmaps (zero features: coordinates 0)."""
    ww, c = W * W, 128
    rs = np.random.RandomState(67)
    u = rs.standard_normal((4, c)).astype(np.float32)
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    f0 = np.zeros((4, ww, c), np.float32)
    f1 = np.zeros((4, ww, c), np.float32)
    # logit gaps 4096 / sqrt(128) = 362 (exactly one-hot in fp32) at three corners, 225 / sqrt(128) = 19.9 off-corner
    peaks, amps = [0, ww - 1, W - 1, ww // 2 + 1], [64.0, 64.0, 64.0, 15.0]
    for m, (p, a) in enumerate(zip(peaks, amps)):
        f0[m, ww // 2] = a * u[m]
        f1[m, p] = a * u[m]
    got, ref = _fine_match(W, f0, f1, 3, f"fine_match_one_hot_W{W}")
    heat_peak = 1.0 / (1.0 + (ww - 1) * np.exp(-(15.0 * 15.0) / np.sqrt(c)))
    assert heat_peak > 1 - 1e-6
    np.testing.assert_array_equal(got[0, :2], [-1, -1])
    np.testing.assert_array_equal(got[1, :2], [1, 1])
    np.testing.assert_array_equal(got[2, :2], [1, -1])
    np.testing.assert_allclose(got[:3, 2], 2e-5, rtol=1e-5)
    np.testing.assert_allclose(ref[:3, 2], 2e-5, rtol=1e-5)
    flat = np.zeros((3, ww, c), np.float32)
    got, ref = _fine_match(W, flat, flat, 5, f"fine_match_flat_W{W}")
    assert np.abs(got[:, :2]).max() < 1e-6 and np.abs(ref[:, :2]).max() < 1e-12


# ------------------------------------------------------------------------------------------------ match all-gather
def test_pack_unpack_matches_single_gpu():
    """pack_matches for three ranks (0, exactly `capacity` and a middle count), stacked, unpack_matches: the CUDA
    kernels against the CPU path of the same functions; a rank over capacity raises OverflowError."""
    from loftr_b200 import parallel
    cap = 96
    rs = np.random.RandomState(71)
    bufs_g, bufs_c = [], []
    offset = 0
    for m in (0, cap, 37):
        d = {"mkpts0_f": torch.from_numpy(rs.uniform(0, 640, (m, 2)).astype(np.float32)),
             "mkpts1_f": torch.from_numpy(rs.uniform(0, 640, (m, 2)).astype(np.float32)),
             "mconf": torch.from_numpy(rs.uniform(0, 1, m).astype(np.float32)),
             "m_bids": torch.from_numpy(np.sort(rs.randint(0, 3, m)).astype(np.int64))}
        bc = parallel.pack_matches(d, offset, cap)
        bg = parallel.pack_matches({k: v.to(DEV) for k, v in d.items()}, offset, cap)
        assert bg.is_cuda and bg.shape == bc.shape == (1 + cap, 6)
        assert torch.equal(bg[: 1 + m].cpu(), bc[: 1 + m]), f"pack m={m}"
        bufs_g.append(bg)
        bufs_c.append(bc)
        offset += 3
    gathered = torch.stack(bufs_g)
    ug = parallel.unpack_matches(gathered)
    uc = parallel.unpack_matches(torch.stack(bufs_c))
    assert ug["counts"] == uc["counts"] == [0, cap, 37]
    for k in ("mkpts0_f", "mkpts1_f", "mconf", "m_bids"):
        assert torch.equal(ug[k].cpu(), uc[k]), k
    assert ug["m_bids"].dtype == torch.int64 and int(ug["m_bids"].min()) >= 3
    over = gathered.clone()
    over[2, 0, 0] = cap + 1
    with pytest.raises(OverflowError):
        parallel.unpack_matches(over)
    too_many = {k: torch.cat([v, v[:1]]) for k, v in ug.items() if k != "counts"}
    with pytest.raises(RuntimeError, match="exceed the gather capacity"):
        parallel.pack_matches(too_many, 0, cap)


# ------------------------------------------------------------------------------------------------ end to end
def _e2e_vs_ref64(model, case, name, min_matches):
    """Engine forward against ref64.hot_path on the PyTorch backbone's features, one pair at a time."""
    inp = build_inputs(case)
    data = {k: _t(v) for k, v in inp.items()}
    model(data)
    got = {k: _np(data[k]) for k in ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f")}
    keys = ["b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f"]
    parts, rows, cols = {k: [] for k in keys}, [], []
    opt = lambda k, b: inp[k][b:b + 1] if k in inp else None
    for b in range(case["n"]):
        with torch.no_grad():
            i0, i1 = _t(inp["image0"][b:b + 1]), _t(inp["image1"][b:b + 1])
            (c0, f0), (c1, f1) = model.backbone(i0), model.backbone(i1)
            out = R.hot_path(model, c0.double(), c1.double(), f0.double(), f1.double(), inp["image0"].shape[2:],
                             opt("mask0", b), opt("mask1", b), opt("scale0", b), opt("scale1", b))
        for k in keys:
            parts[k].append(_np(out[k] + b if k == "b_ids" else out[k]))
        r, c = R.top2(out["conf_matrix"])
        rows.append(_np(r[0]))
        cols.append(_np(c[0]))
        del out
    ref = {k: np.concatenate(v, 0) for k, v in parts.items()}
    gold = {"row_top2_f64": np.stack(rows), "col_top2_f64": np.stack(cols)}
    assert len(ref["b_ids"]) > min_matches, f"{name}: only {len(ref['b_ids'])} reference matches"
    stats = util.compare_matches(got, ref, gold, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995, label=name)
    util.record(name, stats)
    return data, ref


def test_outdoor_ot_832_masked_vs_f64():
    """The shipped outdoor_ot configuration: Sinkhorn with MegaDepth padding masks and scales, 4 pairs at 832 x 832."""
    case = dict(BASELINE_CASES["out4"], name="out4_ot", match_type="sinkhorn")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, _, _ = util.build_model(case, DEV)
    data, _ = _e2e_vs_ref64(model, case, "e2e_out4_ot_832_vs_f64", 4 * 100)
    b, i, j = (_np(data[k]) for k in ("b_ids", "i_ids", "j_ids"))
    for p in range(4):   # nothing from the padded area or its border
        (vh0, vw0), (vh1, vw1) = case["valid0"][p], case["valid1"][p]
        sel = b == p
        assert (i[sel] // 104 < vh0 // 8 - 2).all() and (i[sel] % 104 < vw0 // 8 - 2).all()
        assert (j[sel] // 104 < vh1 // 8 - 2).all() and (j[sel] % 104 < vw1 // 8 - 2).all()


@pytest.mark.parametrize("case", EDGE_CASES, ids=[c["name"] for c in EDGE_CASES])
def test_edge_config_end_to_end_matches_reference_golden(case):
    """fine_window_size = 3 end to end at 96 x 128 (9-row windows, grid step 2 / (W - 1) = 1, W // 2 = 1) against the
    reference's outputs, adjudicated by its float64 run."""
    import loftr_b200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    gold = util.load_golden(case["name"])
    cfg = build_edge_cfg(case)
    model = loftr_b200.LoFTR(cfg).eval()
    state = WT.make_state({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=0)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    model = model.to(DEV)
    data = {k: _t(v) for k, v in build_inputs(case).items()}
    model(data)
    assert data["W"] == case["fine_window_size"]
    got = {k: _np(data[k]) for k in ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f")}
    stats = util.compare_matches(got, gold, gold, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995, label=case["name"])
    m = len(gold["b_ids"])
    assert m > 20 and stats["n"] >= m - max(1, int(0.005 * m))
    util.record("e2e_golden_" + case["name"], stats)
