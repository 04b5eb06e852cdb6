"""Per-pair match cap (`match_coarse.max_matches_per_pair`, `match_cap_kernel`) on every public path.

The cap clears flags between the flag pass and the ordered compaction, and every stage after it is row-local, so each
list key of a capped forward must equal the same rows of the uncapped forward bit for bit (torch.equal), selected in
torch by `match_cap_ref.apply_cap`: per pair, the k largest mconf, ties to the smaller row index i."""
import numpy as np
import pytest
import torch

import loftr_b200
import util
from cases import BASELINE_CASES, CASES, CM_CASES, build_cfg, build_cm_inputs, build_inputs
from loftr_b200 import _lib
from match_cap_ref import LIST_KEYS, apply_cap, capped_rows, per_pair_counts

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_CASE = {c["name"]: c for c in CASES}
_SCALAR_KEYS = ("bs", "hw0_i", "hw1_i", "hw0_c", "hw1_c", "hw0_f", "hw1_f", "W")
_SMALL = {"n": 2, "hw0": (240, 320), "hw1": (240, 320), "thr": 0.0, "images": "smooth"}

GRID = {
    # the cases of tests/test_static_gpu.py
    "b8_640x480_ds_thr0": BASELINE_CASES["b8"],
    "b8_640x480_ds_thr0.2": BASELINE_CASES["b8thr"],
    "b8_640x480_sinkhorn": BASELINE_CASES["b8ot"],
    "b4_832_masked_scaled": BASELINE_CASES["out4"],
    "unequal": _CASE["ds_unequal"],
    "golden_ds_thr0": _CASE["ds_thr0"],
    # full attention in both transformers, and thr < 0 (the mconf != 0 filter runs after the cap)
    "full_attention": dict(_SMALL, name="fa", coarse_attention="full", fine_attention="full"),
    "thr_negative": dict(_SMALL, name="neg", thr=-1.0),
    # pair 1's valid region lies inside the removed border: a pair without matches between two with matches
    "empty_pair": dict(_SMALL, name="empty", n=3, valid0=[(240, 320), (32, 32), (240, 320)],
                       valid1=[(240, 320), (240, 320), (176, 320)]),
    # n = 1 at the largest size (L = 19,200)
    "n1_1280x960": BASELINE_CASES["sweep960"],
}


def _eager(model, inp, k="keep"):
    if k != "keep":
        model.coarse_matching.max_matches_per_pair = k
    data = dict(inp)
    model(data)
    return data


def _assert_capped(got, uncapped, k, label):
    ref = apply_cap(uncapped, k)
    for key in LIST_KEYS:
        assert got[key].dtype == ref[key].dtype, (label, key)
        assert torch.equal(got[key], ref[key]), f"{label}: {key} differs from the selected uncapped rows"
    for key in _SCALAR_KEYS:
        assert got[key] == uncapped[key], (label, key)
    assert got["mkpts0_f"] is got["mkpts0_c"]
    n = uncapped["bs"]
    want = [min(c, k) for c in per_pair_counts(uncapped["b_ids"], n)]
    assert per_pair_counts(got["b_ids"], n) == want, label


def _k_values(counts, L):
    """1, 7, a value below the median count, one pair's exact count and that count - 1, the largest count, L and a
    value past the range of a C int."""
    live = sorted(c for c in counts if c > 0) or [1]
    one = live[len(live) // 2]
    return sorted({1, 7, max(1, int(np.median(counts)) // 2), one, max(1, one - 1), max(live), L, 2 ** 40})


@pytest.mark.parametrize("name", list(GRID))
def test_cap_selects_the_most_confident_rows(name):
    case = GRID[name]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    lib = _lib.load()
    _eager(model, inp, None)   # the first call also packs the weights
    n0 = lib.lb_launch_count()
    uncapped = _eager(model, inp, None)
    launches = lib.lb_launch_count() - n0
    n, L, S = case["n"], int(np.prod(uncapped["hw0_c"])), int(np.prod(uncapped["hw1_c"]))
    counts = per_pair_counts(uncapped["b_ids"], n)
    if name == "empty_pair":
        assert counts[1] == 0 and min(counts[0], counts[2]) > 0, counts
    if case["thr"] == 0.0 and name != "empty_pair":
        assert min(counts) > 0, counts
    masked = "mask0" in inp
    for k in _k_values(counts, L):
        label = f"{name} k={k}"
        n0 = lib.lb_launch_count()
        got = _eager(model, inp, k)
        if k >= max(counts):   # the same list: the select kernel is the one extra launch
            assert lib.lb_launch_count() - n0 == launches + 1, label
        _assert_capped(got, uncapped, k, label)
        if case["thr"] < 0:
            continue   # forward_static refuses thr < 0
        st = dict(inp)
        model.forward_static(st)
        cap = n * min(k, L if masked else min(L, S))
        m = int(st["num_matches"].item())
        assert st["b_ids"].shape == (cap,) and m == got["b_ids"].shape[0] and m <= cap, label
        for key in LIST_KEYS:
            assert torch.equal(st[key][:m], got[key]), f"{label}: static {key} differs from the capped eager run"
    again = _eager(model, inp, None)   # no cap: the uncapped result again
    for key in LIST_KEYS:
        assert torch.equal(again[key], uncapped[key]), key


def test_ties_at_the_kth_value_go_to_the_smaller_row():
    """At a tiny softmax temperature most mutual matches score exactly 1.0 in fp32."""
    case = dict(_SMALL, name="ties")
    model, _, _ = util.build_model(case, DEV)
    model.coarse_matching.temperature = 1e-4
    inp = util.device_inputs(case)
    uncapped = _eager(model, inp, None)
    b_ids, conf, i_ids = uncapped["b_ids"], uncapped["mconf"], uncapped["i_ids"]
    above = [int(((b_ids == b) & (conf > 1.0)).sum()) for b in range(case["n"])]
    ones = [int(((b_ids == b) & (conf == 1.0)).sum()) for b in range(case["n"])]
    assert min(ones) >= 8, f"too few exact ties at 1.0: {ones}"
    cut = 0
    for k in (1, above[0] + ones[0] // 2, above[1] + ones[1] - 1, above[0] + ones[0] + 3):
        got = _eager(model, inp, k)
        _assert_capped(got, uncapped, k, f"ties k={k}")
        for b in range(case["n"]):
            if above[b] < k < above[b] + ones[b]:   # the k-th value is 1.0 and the cap cuts its tie
                kept = got["i_ids"][(got["b_ids"] == b) & (got["mconf"] == 1.0)]
                tied = i_ids[(b_ids == b) & (conf == 1.0)]
                assert torch.equal(kept, tied[:k - above[b]]), (k, b)   # the smallest row indices of the tie
                cut += 1
    assert cut >= 3, "the ties were never cut"


def test_captured_matcher_with_a_cap():
    case = BASELINE_CASES["b8"]
    model, _, _ = util.build_model(case, DEV)
    batches = [util.device_inputs(case, seed) for seed in (1, 2)]
    model.coarse_matching.max_matches_per_pair = 300
    cm = loftr_b200.CapturedMatcher(model, case["n"], case["hw0"])
    assert cm.capacity == 8 * 300

    def check(k):
        for inp in batches:
            got = dict(inp)
            cm(got)
            ref = _eager(model, inp)
            assert set(got) == set(ref)
            for key, v in ref.items():
                if torch.is_tensor(v):
                    assert got[key].shape == v.shape and torch.equal(got[key], v), (k, key)
                else:
                    assert got[key] == v, (k, key)
            if k is not None:
                assert max(per_pair_counts(got["b_ids"], case["n"])) == k

    check(300)
    model.coarse_matching.max_matches_per_pair = 100
    with pytest.raises(RuntimeError, match=r"max_matches_per_pair changed since capture \(300 -> 100\)"):
        cm(dict(batches[0]))
    cm.recapture()
    assert cm.capacity == 8 * 100
    check(100)
    model.coarse_matching.max_matches_per_pair = None
    with pytest.raises(RuntimeError, match="max_matches_per_pair changed since capture"):
        cm(dict(batches[0]))
    cm.recapture()
    assert cm.capacity == 8 * 4800
    check(None)


def test_match_features_equals_capped_matcher_batch():
    """Tensor-core backbone: the bank path and matcher(batch) on the stacked pairs agree bit for bit under a cap."""
    model, _, _ = util.build_model(dict(_SMALL, name="bank"), DEV, "b200")
    inp = build_inputs({"n": 3, "hw0": (480, 640), "hw1": (480, 640), "images": "smooth", "iseed": 1})
    imgs = torch.from_numpy(np.concatenate([inp["image0"], inp["image1"]])).to(DEV)
    bank = model.extract_features(imgs)
    idx0 = torch.tensor([0, 1, 2, 2, 3, 4, 5], device=DEV)
    idx1 = torch.tensor([1, 0, 3, 3, 3, 5, 2], device=DEV)
    for k in (1, 50, 400, None):
        model.coarse_matching.max_matches_per_pair = k
        got = model.match_features(bank, idx0, bank, idx1)
        ref = {"image0": imgs[idx0], "image1": imgs[idx1]}
        model(ref)
        del ref["image0"], ref["image1"]
        assert list(got) == list(ref), k
        for key, v in ref.items():
            if torch.is_tensor(v):
                assert got[key].dtype == v.dtype and torch.equal(got[key], v), (k, key)
            else:
                assert got[key] == v, (k, key)
        if k is not None:
            assert max(per_pair_counts(got["b_ids"], 7)) == k


def test_coarse_matching_module_forward_with_a_cap():
    """The reference-signature CoarseMatching.forward, with conf_matrix: the matrix stays the full one."""
    import loftr_b200.loftr as LL
    case = CM_CASES[0]
    cfg = dict(build_cfg(case)["match_coarse"], return_conf_matrix=True, thr=0.0)
    inp = build_cm_inputs(case)
    f0, f1 = (torch.from_numpy(inp[k]).to(DEV) for k in ("feat_c0", "feat_c1"))
    (h0, w0), (h1, w1) = case["hw0c"], case["hw1c"]

    def run(k):
        mod = LL.CoarseMatching(dict(cfg, max_matches_per_pair=k)).eval()
        data = {"hw0_i": (h0 * 8, w0 * 8), "hw1_i": (h1 * 8, w1 * 8), "hw0_c": (h0, w0), "hw1_c": (h1, w1)}
        mod(f0, f1, data)
        return data

    uncapped = run(None)
    counts = per_pair_counts(uncapped["b_ids"], case["n"])
    assert min(counts) > 10
    for k in (1, 5, min(counts), max(counts) + 1):
        got = run(k)
        idx = capped_rows(uncapped["b_ids"], uncapped["mconf"], k)
        for key in ("b_ids", "i_ids", "j_ids", "m_bids", "gt_mask", "mconf", "mkpts0_c", "mkpts1_c"):
            assert torch.equal(got[key], uncapped[key][idx]), (k, key)
        assert torch.equal(got["conf_matrix"], uncapped["conf_matrix"]), k
