"""Full (softmax) attention in the coarse and fine transformers on the H100, against the reference's goldens and the
numpy oracle (tests/full_oracle.py) under the project's parity rule (`util.compare_matches`): overlap >= 99.5 % by
(b, i, j), every non-shared match an fp64 near-tie, mconf rtol 1e-3, |dxy| < 0.5 px."""
import numpy as np
import pytest
import torch

import full_oracle as FO
import loftr_b200
import util
import weights as W
from cases import build_inputs
from full_cases import FULL_BASELINE_CASES, FULL_CASES, build_full_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_LIST_KEYS = ["b_ids", "i_ids", "j_ids", "m_bids", "gt_mask", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f",
              "expec_f"]
COMBOS = [("linear", "linear"), ("full", "linear"), ("linear", "full"), ("full", "full")]


def _model(case, device=DEV):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = build_full_cfg(case)
    model = loftr_b200.LoFTR(cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    state = W.make_state(shapes, seed=case.get("wseed", 0))
    model.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    return model.to(device), cfg, state


def _inputs(case, seed=None):
    if seed is not None:
        case = dict(case, iseed=seed)
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in build_inputs(case).items()}


def _eager(model, inp):
    data = dict(inp)
    model(data)
    return data


def _np(data):
    return {k: v.cpu().numpy() for k, v in data.items() if torch.is_tensor(v)}


@pytest.mark.parametrize("case", FULL_CASES, ids=[c["name"] for c in FULL_CASES])
def test_full_attention_golden_end_to_end(case):
    gold = util.load_golden(case["name"])
    model, _, _ = _model(case)
    got = _np(_eager(model, _inputs(case)))
    stats = util.compare_matches(got, gold, gold, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995, label=case["name"])
    assert stats["n"] > 0
    util.record("full_attention_golden_" + case["name"], stats)


@pytest.mark.parametrize("which", ["coarse", "fine"])
def test_local_feature_transformer_vs_oracle(which):
    """One transformer alone: L != S, a partial last query tile, padding masks on both sides."""
    case = {"name": "tf", "n": 2, "hw0": (96, 128), "hw1": (96, 128), "coarse_attention": "full",
            "fine_attention": "full"}
    model, cfg, state = _model(case)
    tf = model.loftr_coarse if which == "coarse" else model.loftr_fine
    c = cfg[which]
    rs = np.random.RandomState(3)
    n, L, S = (2, 203, 150) if which == "coarse" else (7, 25, 25)
    f0 = rs.standard_normal((n, L, c["d_model"])).astype(np.float32)
    f1 = rs.standard_normal((n, S, c["d_model"])).astype(np.float32)
    m0 = np.ones((n, L), bool)
    m1 = np.ones((n, S), bool)
    m0[1, 170:] = False
    m1[0, 97:] = False
    m1[1, :11] = False
    t = lambda a: torch.from_numpy(a).to(DEV)
    g0, g1 = tf(t(f0), t(f1), t(m0), t(m1))
    layers = FO.O.split_layers(state, "loftr_" + which, len(c["layer_names"]))
    o0, o1 = FO.local_feature_transformer(f0, f1, layers, c["layer_names"], c["nhead"], m0, m1, "full")
    g0, g1 = g0.cpu().numpy(), g1.cpu().numpy()
    assert np.isfinite(g0).all() and np.isfinite(g1).all()
    np.testing.assert_allclose(g0, o0, rtol=1e-3, atol=1e-3)
    np.testing.assert_allclose(g1, o1, rtol=1e-3, atol=1e-3)
    util.record(f"full_attention_tf_{which}", {"max_abs": float(max(np.abs(g0 - o0).max(), np.abs(g1 - o1).max()))})


def test_full_attention_640x480_vs_oracle():
    case = FULL_BASELINE_CASES["full_b2_640x480"]
    model, _, _ = _model(case)
    got = _np(_eager(model, _inputs(case)))
    ref, gold = FO.oracle_forward_per_pair(case)
    stats = util.compare_matches(got, ref, gold, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995, label=case["name"])
    assert stats["n"] > 500
    util.record("full_attention_640x480_vs_oracle", stats)


def test_full_attention_masked_scaled_vs_oracle():
    """Different valid regions per image (padded queries and keys) and scales: no NaN reaches any output."""
    case = FULL_BASELINE_CASES["full_masked"]
    model, _, _ = _model(case)
    data = _eager(model, _inputs(case))
    for k, v in data.items():
        if torch.is_tensor(v) and v.is_floating_point():
            assert torch.isfinite(v).all(), k
    ref, gold = FO.oracle_forward_per_pair(case)
    stats = util.compare_matches(_np(data), ref, gold, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995,
                                 label=case["name"])
    assert stats["n"] > 100
    util.record("full_attention_masked_scaled_vs_oracle", stats)


def _assert_static_equals_eager(st, eager, label):
    m = int(st["num_matches"].item())
    assert m == eager["b_ids"].shape[0], f"{label}: count {m} vs eager {eager['b_ids'].shape[0]}"
    for k in _LIST_KEYS:
        assert torch.equal(st[k][:m], eager[k]), f"{label}: {k} differs from the eager forward"


@pytest.mark.parametrize("combo", COMBOS, ids=["-".join(c) for c in COMBOS])
def test_forward_static_and_captured_match_eager(combo):
    case = {"name": "combo", "n": 2, "hw0": (96, 128), "hw1": (96, 128), "thr": 0.0, "images": "smooth",
            "coarse_attention": combo[0], "fine_attention": combo[1]}
    model, _, _ = _model(case)
    inp = _inputs(case)
    eager = _eager(model, inp)
    assert eager["b_ids"].shape[0] > 0
    st = dict(inp)
    model.forward_static(st)
    _assert_static_equals_eager(st, eager, f"static {combo}")
    cm = loftr_b200.CapturedMatcher(model, 2, (96, 128))
    for seed in (1, 2):
        batch = _inputs(case, seed)
        ref = _eager(model, batch)
        res = dict(batch)
        cm(res)
        for k in _LIST_KEYS:
            assert torch.equal(res[k], ref[k]), f"captured {combo} seed {seed}: {k}"
    model.coarse_matching.thr = 1.0          # conf > 1 never holds: M = 0
    cm0 = loftr_b200.CapturedMatcher(model, 2, (96, 128))
    ref = _eager(model, inp)
    res = dict(inp)
    cm0(res)
    assert ref["b_ids"].shape[0] == 0 and res["b_ids"].shape[0] == 0
    for k in _LIST_KEYS:
        assert torch.equal(res[k], ref[k]), f"captured {combo} M=0: {k}"


def test_full_attention_is_deterministic():
    case = {"name": "det", "n": 2, "hw0": (480, 640), "hw1": (480, 640), "thr": 0.0, "images": "smooth",
            "coarse_attention": "full", "fine_attention": "full"}
    model, _, _ = _model(case)
    model.expose_coarse_features = True
    inp = _inputs(case)
    a, b = _eager(model, inp), _eager(model, inp)
    for k in _LIST_KEYS + ["_feat_c0", "_feat_c1"]:
        assert torch.equal(a[k], b[k]), k
