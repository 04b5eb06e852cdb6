"""The rectification search (data["rectify1_candidates"], `rotation_candidates`, lb_coarse_match_search; DESIGN.md §20)
on the GPU:
1. equivalence: the search equals the rectified forward on the N * K candidate pairs restricted to each pair's chosen
   candidate, bit for bit in every list key and minside1 (split and fp16, dual-softmax and Sinkhorn, with and without a
   per-pair cap, with masks and scales); rectify1_counts are that forward's uncapped per-candidate match counts and
   rectify1_choice the reference's choice;
2. ties from duplicate candidates go to the smaller k;
3. K = 1 is the rectify1 call bit for bit, and identity candidates with equal sizes and scales the plain call;
4. `warp_images` of torch.rot90(image, q) through candidate q of `rotation_candidates` is the image bit for bit;
5. a pair's outputs do not depend on the other pairs' candidates, a NaN candidate acts as the identity, and a pair
   with no match under any candidate gets choice 0 and no matches;
6. forward_static matches the eager call within the N-pair default capacity, and a CUDA graph follows the candidate
   tensor from replay to replay."""
import numpy as np
import pytest
import torch

import loftr_b200
import rectify_search_ref as SR
import util
from cases import CASES
from loftr_b200.loftr import CoarseMatching
from match_cap_ref import LIST_KEYS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_CASE = {c["name"]: c for c in CASES}
INPUTS = util.INPUT_KEYS + ("rectify1", "rectify1_candidates")
SEARCH_KEYS = ("rectify1_choice", "rectify1_counts")
KEYS = LIST_KEYS + ["minside1"]


def _candidates(inp, params):
    """[N, K, 3, 3] float32 on the device: per pair, one similarity about the image centres (source pixels) per
    (degrees, zoom) of `params`."""
    n, hw0, hw1 = inp["image0"].shape[0], inp["image0"].shape[2:], inp["image1"].shape[2:]
    s0 = inp["scale0"].cpu().numpy() if "scale0" in inp else np.ones((n, 2))
    s1 = inp["scale1"].cpu().numpy() if "scale1" in inp else np.ones((n, 2))
    c = [[util.similarity((0.5 * (hw0[1] - 1) * s0[b, 0], 0.5 * (hw0[0] - 1) * s0[b, 1]),
                          (0.5 * (hw1[1] - 1) * s1[b, 0], 0.5 * (hw1[0] - 1) * s1[b, 1]), deg + 3 * b, zoom)
          for deg, zoom in params] for b in range(n)]
    return torch.from_numpy(np.array(c)).float().to(DEV)


def _flattened(inp, cands):
    """The rectified forward's input on the N * K candidate pairs: candidate c = b * K + k has pair b's images, masks
    and scales and rectify1 = cands[b, k]."""
    n, k = cands.shape[:2]
    d = {key: v.repeat_interleave(k, 0) for key, v in inp.items()}
    d["rectify1"] = cands.reshape(n * k, 3, 3)
    return d


def _check_search(model, inp, cands, label):
    """The search on `inp` against the flattened rectified forward -> the search's outputs."""
    n, k = cands.shape[:2]
    got = util.eager(model, dict(inp, rectify1_candidates=cands))
    flat = util.eager(model, _flattened(inp, cands))
    cap = model.coarse_matching.max_matches_per_pair
    model.coarse_matching.max_matches_per_pair = None
    uncapped = flat if cap is None else util.eager(model, _flattened(inp, cands))
    model.coarse_matching.max_matches_per_pair = cap
    counts = SR.counts_from_ids(uncapped["b_ids"], n, k)
    choice = SR.choose(counts)
    assert got["rectify1_counts"].dtype == torch.int32 and got["rectify1_choice"].dtype == torch.int64
    assert np.array_equal(got["rectify1_counts"].cpu().numpy(), counts), label
    assert np.array_equal(got["rectify1_choice"].cpu().numpy(), choice), label
    util.assert_same(got, SR.winners(flat, choice, k, KEYS), KEYS, label)
    assert got["bs"] == n and got["m_bids"] is got["b_ids"]
    for key in INPUTS:   # the caller's inputs are not replaced
        if key in inp:
            assert got[key] is inp[key], key
    return got, counts


# ------------------------------------------------------------------------------------------------ 1. equivalence
EQUIV = [("ds_thr0", "split", None), ("ds_thr0", "fp16", 12), ("ot_thr0", "split", 9),
         ("ds_masked_scaled", "split", 7), ("ot_masked", "fp16", None)]


@pytest.mark.parametrize("name, precision, cap", EQUIV, ids=[f"{a}_{b}_cap{c}" for a, b, c in EQUIV])
def test_search_is_the_flattened_forward_restricted_to_the_winners(name, precision, cap):
    case = _CASE[name]
    model, _, _ = util.build_model(case, DEV, match_precision=precision)
    model.coarse_matching.max_matches_per_pair = cap
    inp = util.device_inputs(case)
    cands = _candidates(inp, [(75, 1.0), (4, 1.05), (25, 0.85)])
    got, counts = _check_search(model, inp, cands, name)
    assert got["b_ids"].numel() > 0 and len(set(counts.flatten().tolist())) > 1
    if cap is not None:
        assert int(torch.bincount(got["b_ids"]).max()) <= cap
        assert counts.max() > cap   # the cap acts on the winner
    util.record(f"rectify_search_{name}_{precision}_cap{cap}", {"counts": counts.tolist(),
                                                                "matches": int(got["b_ids"].numel())})


# ------------------------------------------------------------------------------------------------ 2. ties
def test_duplicate_candidates_tie_to_the_smaller_k():
    case = _CASE["ds_masked_scaled"]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    cands = _candidates(inp, [(40, 1.0), (3, 1.0), (40, 1.0), (3, 1.0)])   # k and k + 2 are the same model
    got, counts = _check_search(model, inp, cands, "ties")
    assert np.array_equal(counts[:, :2], counts[:, 2:])
    assert set(got["rectify1_choice"].tolist()) <= {0, 1}


# ------------------------------------------------------------------------------------------------ 3. K = 1
@pytest.mark.parametrize("name, precision, cap", [("ds_thr0", "split", None), ("ds_masked_scaled", "fp16", 7)])
def test_one_candidate_is_the_rectified_call(name, precision, cap):
    case = _CASE[name]
    model, _, _ = util.build_model(case, DEV, match_precision=precision)
    model.coarse_matching.max_matches_per_pair = cap
    inp = util.device_inputs(case)
    cands = _candidates(inp, [(12, 0.95)])
    got = util.eager(model, dict(inp, rectify1_candidates=cands))
    ref = util.eager(model, dict(inp, rectify1=cands[:, 0].contiguous()))
    assert ref["b_ids"].numel() > 0
    util.assert_same(got, util.outputs(ref, INPUTS), label=f"{name} K=1")
    assert (got["rectify1_choice"] == 0).all()
    assert got["rectify1_counts"].shape == (inp["image0"].shape[0], 1)
    # identity candidates with equal sizes, scales and masks: the plain call
    if "scale0" in inp:
        inp["scale1"] = inp["scale0"].clone()
    if "mask0" in inp:
        inp["mask1"] = inp["mask0"].clone()
    plain = util.eager(model, inp)
    eye = torch.eye(3, device=DEV).repeat(inp["image0"].shape[0], 1, 1, 1)
    got = util.eager(model, dict(inp, rectify1_candidates=eye))
    util.assert_same(got, util.outputs(plain, INPUTS), label=f"{name} identity")


# ------------------------------------------------------------------------------------------------ 4. quarter turns
@pytest.mark.parametrize("hw", [(64, 64), (48, 80)])
def test_rotation_candidates_undo_rot90_bit_for_bit(hw):
    h, w = hw
    img = torch.rand(2, 1, h, w, generator=torch.Generator().manual_seed(5)).to(DEV)
    size0 = torch.tensor([[w, h]] * 2, dtype=torch.int32, device=DEV)
    for q in range(4):
        rot = torch.rot90(img, q, dims=(-2, -1)).contiguous()
        size1 = torch.tensor([[rot.shape[3], rot.shape[2]]] * 2, dtype=torch.int32, device=DEV)
        cands = loftr_b200.rotation_candidates(size0, size1)
        assert cands.shape == (2, 4, 3, 3) and cands.device == img.device
        back = loftr_b200.warp_images(rot, cands[:, q].contiguous(), (h, w))
        assert torch.equal(back, img), (hw, q)


# ------------------------------------------------------------------------------------------------ 5. per pair, edges
def test_pairs_are_independent_nan_is_the_identity_and_empty_pairs_choose_0():
    case = _CASE["ds_thr0"]
    model, _, _ = util.build_model(case, DEV)
    inp = util.device_inputs(case)
    a = _candidates(inp, [(60, 1.0), (0, 1.0), (20, 1.1)])
    b = a.clone()
    b[1] = _candidates(inp, [(-35, 0.9), (8, 1.0), (90, 1.0)])[1]
    ra = util.eager(model, dict(inp, rectify1_candidates=a))
    rb = util.eager(model, dict(inp, rectify1_candidates=b))
    sa, sb = ra["b_ids"] == 0, rb["b_ids"] == 0
    assert sa.any()
    util.assert_same({k: ra[k][sa] for k in KEYS}, {k: rb[k][sb] for k in KEYS}, label="pair 0")
    util.assert_same({k: ra[k][0] for k in SEARCH_KEYS}, {k: rb[k][0] for k in SEARCH_KEYS}, label="pair 0")
    assert not util.same(ra["rectify1_counts"][1], rb["rectify1_counts"][1])
    # a candidate with a non-finite entry is the identity
    eye = a.clone()
    eye[:, 1] = torch.eye(3, device=DEV)
    nan = a.clone()
    nan[:, 1] = float("nan")
    ri = util.eager(model, dict(inp, rectify1_candidates=eye))
    rn = util.eager(model, dict(inp, rectify1_candidates=nan))
    util.assert_same(rn, ri, KEYS + list(SEARCH_KEYS), "nan candidate")
    # no match under any candidate: choice 0, zero counts, an empty list
    empty = _CASE["ds_empty"]
    model, _, _ = util.build_model(empty, DEV)
    inp = util.device_inputs(empty)
    ident = torch.eye(3, device=DEV).repeat(1, 3, 1, 1)
    ident[0, 1], ident[0, 2] = float("nan"), -ident[0, 2]
    got = util.eager(model, dict(inp, rectify1_candidates=ident))
    assert got["rectify1_choice"].tolist() == [0] and got["rectify1_counts"].tolist() == [[0, 0, 0]]
    assert all(got[k].shape[0] == 0 for k in KEYS)


# ------------------------------------------------------------------------------------------------ 6. static, graph
def test_forward_static_and_graph_replay_follow_the_candidates():
    case = _CASE["ds_masked_scaled"]
    model, _, _ = util.build_model(case, DEV)
    model.coarse_matching.max_matches_per_pair = 9
    inp = util.device_inputs(case)
    c1 = _candidates(inp, [(30, 1.0), (2, 1.0)])
    c2 = _candidates(inp, [(-6, 1.1), (45, 1.0), (5, 0.95)])[:, :2].contiguous()
    e1 = util.eager(model, dict(inp, rectify1_candidates=c1))
    e2 = util.eager(model, dict(inp, rectify1_candidates=c2))
    assert e1["b_ids"].numel() > 0 and not util.same(e1["rectify1_counts"], e2["rectify1_counts"])
    n, _, h, w = inp["image0"].shape
    L = (h // 8) * (w // 8)

    def check(st, eager, label):
        util.assert_static_equals_eager(st, eager, label)
        m = int(st["num_matches"].item())
        assert torch.equal(st["minside1"][:m], eager["minside1"]), label
        util.assert_same(st, eager, SEARCH_KEYS, label)

    st = dict(inp, rectify1_candidates=c1)
    model.forward_static(st)
    assert st["b_ids"].shape[0] == CoarseMatching.default_capacity(n, L, L, True, 9) == n * 9
    check(st, e1, "forward_static")
    cands = c1.clone()
    model.forward_static(dict(inp, rectify1_candidates=cands))   # eager warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    out = dict(inp, rectify1_candidates=cands)
    with torch.cuda.graph(g):
        model.forward_static(out)
    for label, c, eager in (("candidates 1", c1, e1), ("candidates 2", c2, e2)):
        cands.copy_(c)   # the graph reads the candidates from the same tensor at every replay
        g.replay()
        check(out, eager, f"graph replay, {label}")
