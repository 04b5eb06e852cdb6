"""CPU-side checks of the per-pair match cap (`match_coarse.max_matches_per_pair`): config validation, the library
version guard, the C entry point's argument check and the torch reference selection the GPU tests compare against."""
import ctypes as C

import numpy as np
import pytest
import torch

import loftr_b200
import util
from loftr_b200 import _lib
from loftr_b200.loftr import CoarseMatching
from match_cap_ref import apply_cap, capped_rows


def _mc_cfg(**kw):
    return dict(loftr_b200.get_cfg("indoor_ds")["match_coarse"], **kw)


@pytest.mark.parametrize("k", [1, 7, 4800, 2 ** 40, np.int64(3), None])
def test_valid_caps_are_accepted(k):
    cm = CoarseMatching(_mc_cfg(max_matches_per_pair=k))
    assert cm.max_matches_per_pair == (None if k is None else int(k))
    assert cm.max_matches_per_pair is None or type(cm.max_matches_per_pair) is int
    assert CoarseMatching(_mc_cfg()).max_matches_per_pair is None   # absent key: no cap


@pytest.mark.parametrize("k", [0, -1, 2.0, 2.5, "8", True, False, [4]])
def test_invalid_caps_are_rejected(k):
    with pytest.raises(ValueError, match="max_matches_per_pair"):
        CoarseMatching(_mc_cfg(max_matches_per_pair=k))
    cfg = loftr_b200.get_cfg("indoor_ds")
    cfg["match_coarse"]["max_matches_per_pair"] = k
    with pytest.raises(ValueError, match="max_matches_per_pair"):
        loftr_b200.LoFTR(cfg)
    cm = CoarseMatching(_mc_cfg(max_matches_per_pair=5))
    with pytest.raises(ValueError, match="max_matches_per_pair"):   # the attribute is validated as well
        cm.max_matches_per_pair = k
    assert cm.max_matches_per_pair == 5


def test_default_capacity_with_a_cap():
    dc = CoarseMatching.default_capacity
    assert dc(8, 4800, 4800, False) == 8 * 4800
    assert dc(8, 4800, 4800, False, 256) == 8 * 256
    assert dc(2, 300, 200, False, 250) == 2 * 200    # min(k, min(L, S))
    assert dc(2, 300, 200, True, 250) == 2 * 250     # masked: min(k, L)
    assert dc(2, 300, 200, True, 400) == 2 * 300
    assert dc(0, 300, 200, False, 4) == 1


def test_capped_matching_refuses_an_older_library(monkeypatch):
    util.old_library(monkeypatch, 104)
    assert _lib.MATCH_CAP_VERSION == 105
    cm = CoarseMatching(_mc_cfg(max_matches_per_pair=16)).eval()
    with pytest.raises(RuntimeError, match=r"version 105 or newer.*is version 104"):
        cm.run(None, None, 256, 1, 4, 4, 256, {})
    # without a cap the older library is not what stops the call
    cm.max_matches_per_pair = None
    with pytest.raises(AttributeError):
        cm.run(None, None, 256, 1, 4, 4, 256, {})


def test_capped_entry_point_is_bound_and_checks_k():
    lib = _lib.load()
    assert lib.lb_version() >= _lib.MATCH_CAP_VERSION
    assert _lib.SIGNATURES["lb_coarse_match_capped"][1] == lib.lb_coarse_match_capped.argtypes
    a = _lib.LbCoarseMatchArgs()
    for k in (0, -3):
        assert lib.lb_coarse_match_capped(C.byref(a), k, None, 0, None) != 0
        assert b"max_per_pair must be at least 1" in lib.lb_last_error()


def test_reference_selection_on_hand_made_lists():
    # pair 0: rows with mconf 0.5, 0.9, 0.5, 0.5, 0.1 (a three-way tie at 0.5); pair 1: nothing; pair 2: two rows
    b = torch.tensor([0, 0, 0, 0, 0, 2, 2])
    i = torch.tensor([3, 4, 8, 9, 11, 0, 5])
    conf = torch.tensor([0.5, 0.9, 0.5, 0.5, 0.1, 0.3, 0.3])
    got = lambda k: capped_rows(b, conf, k).tolist()
    assert got(1) == [1, 5]                  # the best of pair 0; the tie in pair 2 goes to the smaller i
    assert got(2) == [0, 1, 5, 6]            # 0.9 + the first 0.5 (i = 3)
    assert got(3) == [0, 1, 2, 5, 6]         # 0.9 + the 0.5 rows at i = 3, 8; not i = 9
    assert got(4) == [0, 1, 2, 3, 5, 6]
    assert got(5) == got(100) == list(range(7))
    assert capped_rows(b[:0], conf[:0], 3).tolist() == []

    out = {"b_ids": b, "i_ids": i, "j_ids": i + 1, "m_bids": b, "gt_mask": torch.zeros(7, dtype=torch.bool),
           "mconf": conf, "mkpts0_c": torch.stack([i, b], 1).float(), "mkpts1_c": torch.stack([b, i], 1).float(),
           "mkpts1_f": torch.rand(7, 2), "expec_f": torch.rand(7, 3)}
    out["mkpts0_f"] = out["mkpts0_c"]
    sub = apply_cap(out, 3)
    assert sub["i_ids"].tolist() == [3, 4, 8, 0, 5] and torch.equal(sub["mconf"], conf[[0, 1, 2, 5, 6]])
    assert torch.equal(sub["expec_f"], out["expec_f"][[0, 1, 2, 5, 6]])
