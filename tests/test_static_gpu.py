"""Sync-free static-shape forward (`LoFTR.forward_static`) and CUDA-graph replay (`loftr_b200.CapturedMatcher`).

Every kernel on the path is deterministic and row-local, and the device-bounded fine stage computes each live window
with the same instructions as the eager forward, so the live prefix of every static output must equal the eager
output bit for bit (torch.equal, no tolerance)."""
import numpy as np
import pytest
import torch

import loftr_b200
import util
from cases import BASELINE_CASES, CASES, build_inputs
from loftr_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_CASE = {c["name"]: c for c in CASES}
# keys of `forward` whose first dimension is the match count
_LIST_KEYS = ["b_ids", "i_ids", "j_ids", "m_bids", "gt_mask", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f",
              "expec_f"]


def _inputs(case, seed=None):
    if seed is not None:
        case = dict(case, iseed=seed)
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in build_inputs(case).items()}


def _model(case, backbone_impl="auto"):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, cfg, _ = util.build_model(case, "cpu")
    if backbone_impl != "auto":
        m2 = loftr_b200.LoFTR(cfg, backbone_impl=backbone_impl).eval()
        m2.load_state_dict(model.state_dict())
        model = m2
    return model.to(DEV)


def _eager(model, inp):
    data = dict(inp)
    model(data)
    return data


def _assert_static_equals_eager(st, eager, label):
    m = int(st["num_matches"].item())
    assert m == eager["b_ids"].shape[0], f"{label}: count {m} vs eager {eager['b_ids'].shape[0]}"
    assert m <= st["b_ids"].shape[0]
    for k in _LIST_KEYS:
        assert st[k].dtype == eager[k].dtype, (label, k)
        assert torch.equal(st[k][:m], eager[k]), f"{label}: {k} differs from the eager forward"
    assert st["mkpts0_f"] is st["mkpts0_c"]
    for k in ("bs", "hw0_i", "hw1_i", "hw0_c", "hw1_c", "hw0_f", "hw1_f", "W"):
        assert st[k] == eager[k], (label, k)


STATIC_CASES = {
    "b8_640x480_ds_thr0": BASELINE_CASES["b8"],
    "b8_640x480_ds_thr0.2": BASELINE_CASES["b8thr"],
    "b8_640x480_sinkhorn": BASELINE_CASES["b8ot"],
    "b4_832_masked_scaled": BASELINE_CASES["out4"],
    "unequal": _CASE["ds_unequal"],
    "golden_ds_thr0": _CASE["ds_thr0"],
}


@pytest.mark.parametrize("name", list(STATIC_CASES))
def test_forward_static_matches_eager_bitwise(name):
    case = STATIC_CASES[name]
    model = _model(case)
    inp = _inputs(case)
    eager = _eager(model, inp)
    st = dict(inp)
    model.forward_static(st)
    _assert_static_equals_eager(st, eager, name)
    n, L, S = case["n"], int(np.prod(eager["hw0_c"])), int(np.prod(eager["hw1_c"]))
    cap = n * L if "mask0" in inp else n * min(L, S)
    assert st["b_ids"].shape == (cap,) and st["expec_f"].shape == (cap, 3)
    assert st["num_matches"].dtype == torch.int32 and st["num_matches"].shape == (1,)
    util.record("static_vs_eager_" + name, {"n": int(st["num_matches"].item()), "capacity": cap})


def test_forward_static_has_no_host_sync_and_captures():
    case = _CASE["ds_thr0"]
    model = _model(case)
    inp = _inputs(case)
    eager = _eager(model, inp)                 # packs the weights (that synchronises once)
    st = dict(inp)
    model.forward_static(st)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        st = dict(inp)
        model.forward_static(st)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _assert_static_equals_eager(st, eager, "no-sync")
    g = torch.cuda.CUDAGraph()
    out = dict(inp)
    with torch.cuda.graph(g):
        model.forward_static(out)
    g.replay()
    _assert_static_equals_eager(out, eager, "graph replay")


def _three_batches(case, model):
    """Three input batches and a threshold under which one gives M = 0 and the other two 0 < M_first < M_last.
    Mutual nearest neighbours do not depend on thr, so M(thr) = #(thr-0 matches with mconf > thr); the batch with the
    lowest top confidence sets thr to exactly that confidence (conf > thr is strict)."""
    batches = [_inputs(case, seed) for seed in (1, 2, 3, 4)]
    model.coarse_matching.thr = 0.0
    confs = [_eager(model, b)["mconf"] for b in batches]
    top = [float(c.max()) if c.numel() else 0.0 for c in confs]
    z = int(np.argmin(top))
    thr = top[z]
    counts = [int((c > thr).sum()) for c in confs]
    others = sorted((i for i in range(len(batches)) if i != z), key=lambda i: counts[i])
    first, last = others[0], others[-1]
    assert counts[first] > 0 and counts[last] > counts[first], f"unusable batches: {counts} at {thr}"
    model.coarse_matching.thr = thr
    return [batches[first], batches[z], batches[last]]


@pytest.mark.parametrize("impl,case", [("b200", BASELINE_CASES["b8"]),
                                       ("torch", dict(_CASE["ds_thr0"], hw0=(240, 320), hw1=(240, 320)))],
                         ids=["b200-b8-640x480", "torch-2x320x240"])
def test_captured_matcher_replays_equal_eager(impl, case):
    model = _model(case, impl)
    batches = _three_batches(case, model)
    cm = loftr_b200.CapturedMatcher(model, case["n"], case["hw0"], case["hw1"])
    results, kept = [], []
    for inp in batches:
        got = dict(inp)
        cm(got)
        ref = _eager(model, inp)
        assert set(got) == set(ref)
        for k, v in ref.items():
            if torch.is_tensor(v):
                assert got[k].shape == v.shape and torch.equal(got[k], v), f"{impl}: {k}"
            else:
                assert got[k] == v, f"{impl}: {k}"
        assert got["m_bids"] is got["b_ids"] and got["mkpts0_f"] is got["mkpts0_c"]
        results.append({k: v.clone() for k, v in got.items() if torch.is_tensor(v)})
        kept.append(got)
    assert [r["b_ids"].shape[0] for r in results][1] == 0
    for snapshot, got in zip(results, kept):        # later replays leave earlier outputs alone
        for k, v in snapshot.items():
            assert torch.equal(got[k], v)


def test_capacity_overflow_is_reported():
    case = _CASE["ds_thr0"]
    model = _model(case)
    inp = _inputs(case)
    m = _eager(model, inp)["b_ids"].shape[0]
    assert m > 2
    st = dict(inp)
    model.forward_static(st, capacity=2)
    assert int(st["num_matches"].item()) == m and st["b_ids"].shape == (2,)
    cm = loftr_b200.CapturedMatcher(model, case["n"], case["hw0"], capacity=2)
    with pytest.raises(RuntimeError, match=rf"{m} coarse matches exceed the capacity 2"):
        cm(dict(inp))


def test_weight_change_after_capture_raises_until_recapture():
    case = _CASE["ds_thr0"]
    model = _model(case)
    inp = _inputs(case)
    cm = loftr_b200.CapturedMatcher(model, case["n"], case["hw0"])
    cm(dict(inp))
    other = _model(dict(case, wseed=5))
    model.load_state_dict(other.state_dict())
    with pytest.raises(RuntimeError, match="weights changed since capture"):
        cm(dict(inp))
    cm.recapture()
    got = dict(inp)
    cm(got)
    ref = _eager(model, inp)
    for k in _LIST_KEYS:
        assert torch.equal(got[k], ref[k]), k
    model.invalidate_packed()
    with pytest.raises(RuntimeError, match="weights changed since capture"):
        cm(dict(inp))


def test_timing_during_capture_fails_loudly():
    case = _CASE["ds_thr0"]
    model = _model(case)
    inp = _inputs(case)
    model.forward_static(dict(inp))
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    _lib.timing_enable(True)
    try:
        with pytest.raises(RuntimeError, match="timing events cannot be recorded into a graph"):
            with torch.cuda.graph(g):
                model.forward_static(dict(inp))
    finally:
        _lib.timing_enable(False)
    del g
