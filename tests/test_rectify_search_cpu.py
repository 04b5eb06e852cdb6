"""CPU-side checks of the rectification search (data["rectify1_candidates"], DESIGN.md §20): the validator and the
callers that refuse the key, the binding of lb_coarse_match_search by name and its argument errors,
`rotation_candidates` against a float64 restatement, and self-checks of the selection reference
(tests/rectify_search_ref.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import loftr_b200
import rectify_search_ref as SR
import util
from loftr_b200 import _lib
from loftr_b200.loftr import CapturedMatcher, check_rectify_candidates


def _cands(n=2, k=4, **kw):
    return torch.eye(3, **kw).repeat(n, k, 1, 1)


@pytest.mark.parametrize("cands, exc, match", [
    (np.eye(3, dtype=np.float32)[None, None].repeat(2, 0), TypeError, "rectify1_candidates must be a float32 tensor"),
    (_cands(dtype=torch.float64), TypeError, "rectify1_candidates must be a float32 tensor"),
    (torch.eye(3).repeat(2, 1, 1), ValueError, r"rectify1_candidates must be \[N, K, 3, 3\] with N = 2"),
    (_cands(3), ValueError, r"rectify1_candidates must be \[N, K, 3, 3\] with N = 2 pairs \(got \(3, 4, 3, 3\)\)"),
    (torch.zeros(2, 4, 9), ValueError, r"rectify1_candidates must be \[N, K, 3, 3\]"),
    (_cands(k=0), ValueError, r"rectify1_candidates needs at least one candidate per pair \(got K = 0\)"),
    (_cands(k=32768), ValueError, r"rectify1_candidates holds N \* K = 65536 candidate pairs, more than the warp's "
                                  "65535"),
    (_cands(device="meta"), ValueError, "rectify1_candidates is on meta, the images on cpu"),
    (_cands(), ValueError, "rectify1_candidates must be a CUDA tensor"),
], ids=["numpy", "f64", "rank", "n", "shape", "k0", "too_many", "device", "host"])
def test_validator_rejects(cands, exc, match):
    with pytest.raises(exc, match="forward: " + match):
        check_rectify_candidates(cands, 2, torch.device("cpu"), "forward")


def test_validator_accepts_the_largest_batch_up_to_the_device_check():
    with pytest.raises(ValueError, match="must be a CUDA tensor"):   # 65535 candidate pairs pass the count check
        check_rectify_candidates(_cands(1, 65535), 1, torch.device("cpu"), "forward")


def _model():
    return loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).eval()


def test_search_refuses_rectify1_and_a_guide_before_any_launch():
    m = _model()
    base = {"image0": torch.zeros(1, 1, 8, 8), "image1": torch.zeros(1, 1, 8, 8), "rectify1_candidates": _cands(1)}
    guide = {"kind": "homography", "model": torch.eye(3)[None], "radius": 8.0}
    for who in ("forward", "forward_static"):
        with pytest.raises(ValueError, match=rf"{who}: data\['rectify1_candidates'\] cannot be combined with "
                                             r"data\['rectify1'\]"):
            m._match_searched(dict(base, rectify1=torch.eye(3)[None]), who)
        with pytest.raises(ValueError, match=rf"{who}: data\['rectify1_candidates'\] cannot be combined with "
                                             r"data\['guide'\]"):
            m._match_searched(dict(base, guide=guide), who)
    with pytest.raises(ValueError, match="forward: rectify1_candidates must be a CUDA tensor"):
        m._match_searched(base, "forward")


def test_match_points_and_the_captured_matcher_refuse_the_key():
    m = _model()
    data = {"image0": torch.zeros(1, 1, 8, 8), "image1": torch.zeros(1, 1, 8, 8), "rectify1_candidates": _cands(1)}
    with pytest.raises(ValueError, match=r"match_points: data\['rectify1_candidates'\] is not supported"):
        m.match_points(data, torch.zeros(1, 4, 2))
    cap = CapturedMatcher.__new__(CapturedMatcher)   # refused before the graph or the weights are read
    cap.graph = None
    with pytest.raises(ValueError, match=r"CapturedMatcher: data\['rectify1_candidates'\] is not supported"):
        cap({"image0": torch.zeros(1, 1, 8, 8), "rectify1_candidates": _cands(1)})


def test_search_entry_is_bound_only_where_exported(monkeypatch):
    """lb_coarse_match_search comes without a version step, found by name like the rectify entries: the shipped build
    exports and binds it; a build without it still loads, and only the search is refused."""
    lib = _lib.load()
    assert _lib.SEARCH_ENTRIES == ("lb_coarse_match_search",)
    name = "lb_coarse_match_search"
    assert name not in _lib._SINCE and name in _lib._OPTIONAL
    assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    assert lib.lb_version() == 110
    _lib.require_entries(_lib.SEARCH_ENTRIES, "the rectification search")
    names = {lib.lb_timing_tag_name(i).decode() for i in range(lib.lb_timing_num_tags())}
    assert {"match_search", "match_cap", "rectify"} <= names
    old = util.load_without(monkeypatch, _lib.SEARCH_ENTRIES)
    assert not hasattr(old, name)
    assert old.lb_rectify_images.argtypes == _lib.SIGNATURES["lb_rectify_images"][1]   # the rest still binds
    _lib.require_entries(_lib.RECTIFY_ENTRIES + _lib.GUIDE_ENTRIES, "other paths")
    with pytest.raises(RuntimeError, match=r"forward: the rectification search needs lb_coarse_match_search.*"
                                           r"\(version 110\)"):
        check_rectify_candidates(_cands(), 2, torch.device("cpu"), "forward")


def test_search_entry_checks_its_arguments():
    lib = _lib.load()
    buf = torch.zeros(64)
    p = buf.data_ptr()
    a = _lib.LbCoarseMatchArgs()
    a.n_pairs, a.L, a.S = 8, 4, 4
    cases = [(None, 0, 0, b"the search and its counts and choice outputs are required"),
             (_lib.LbCoarseSearch(4, None, p), 0, 0, b"counts and choice outputs are required"),
             (_lib.LbCoarseSearch(4, p, None), 0, 0, b"counts and choice outputs are required"),
             (_lib.LbCoarseSearch(0, p, p), 0, 0, b"K=0 must be at least 1"),
             (_lib.LbCoarseSearch(-2, p, p), 0, 0, b"K=-2 must be at least 1"),
             (_lib.LbCoarseSearch(3, p, p), 0, 0, b"n_pairs=8 is not a multiple of K=3"),
             (_lib.LbCoarseSearch(4, p, p), -1, 0, b"max_per_pair must be 0 (no cap) or at least 1 (got -1)"),
             (_lib.LbCoarseSearch(4, p, p), 0, 2, b"fp16 must be 0 (split) or 1 (got 2)")]
    for search, cap, fp16, msg in cases:
        ref = None if search is None else C.byref(search)
        assert lib.lb_coarse_match_search(C.byref(a), ref, cap, fp16, p, 256, None) != 0
        assert msg in lib.lb_last_error(), (msg, lib.lb_last_error())
        assert b"lb_coarse_match_search: " in lib.lb_last_error()


# ------------------------------------------------------------------------------------------------ rotation_candidates
def _restated(size0, size1, scale0=None, scale1=None):
    """H_q = S1 T(c1) R^q T(-c0) S0^-1 in float64 numpy, one explicit matrix product per pair and turn."""
    n = len(size0)
    s0 = np.ones((n, 2)) if scale0 is None else np.asarray(scale0, np.float64)
    s1 = np.ones((n, 2)) if scale1 is None else np.asarray(scale1, np.float64)
    r1 = np.array([[0.0, 1, 0], [-1, 0, 0], [0, 0, 1]])
    out = np.zeros((n, 4, 3, 3))
    for b in range(n):
        c0 = (np.asarray(size0[b], np.float64) - 1) / 2
        c1 = (np.asarray(size1[b], np.float64) - 1) / 2
        t0 = np.array([[1, 0, -c0[0]], [0, 1, -c0[1]], [0, 0, 1]])
        t1 = np.array([[1, 0, c1[0]], [0, 1, c1[1]], [0, 0, 1]])
        for q in range(4):
            out[b, q] = (np.diag([s1[b, 0], s1[b, 1], 1.0]) @ t1 @ np.linalg.matrix_power(r1, q) @ t0
                         @ np.diag([1 / s0[b, 0], 1 / s0[b, 1], 1.0]))
    return out


def test_rotation_candidates_match_the_float64_restatement():
    size0 = torch.tensor([[640, 480], [480, 640], [200, 136], [33, 17]], dtype=torch.int32)
    size1 = torch.tensor([[480, 640], [480, 640], [128, 200], [64, 48]], dtype=torch.int32)
    got = loftr_b200.rotation_candidates(size0, size1)
    assert got.dtype == torch.float32 and got.shape == (4, 4, 3, 3) and got.is_contiguous()
    want = _restated(size0.numpy(), size1.numpy())
    assert torch.equal(got, torch.from_numpy(want.astype(np.float32)))
    assert np.array_equal(want * 2, np.rint(want * 2))   # whole and half pixels: exact in float32
    assert not torch.signbit(got[got == 0]).any()   # no negative zeros
    assert torch.equal(got[:, 0, :2, :2], torch.eye(2).expand(4, 2, 2))
    assert torch.equal(got[:, 1, :2, :2], torch.tensor([[0.0, 1], [-1, 0]]).expand(4, 2, 2))
    rs = np.random.RandomState(3)
    s0, s1 = rs.uniform(0.5, 2.5, (4, 2)).astype(np.float32), rs.uniform(0.5, 2.5, (4, 2)).astype(np.float32)
    got = loftr_b200.rotation_candidates(size0.float(), size1.long(), torch.from_numpy(s0), torch.from_numpy(s1))
    want = _restated(size0.numpy(), size1.numpy(), s0, s1)
    assert torch.equal(got, torch.from_numpy(want.astype(np.float32)))


@pytest.mark.parametrize("hw", [(48, 48), (24, 40)])
def test_rotation_candidates_take_rot90_images_back_pixel_for_pixel(hw):
    """Candidate q maps every pixel of image0 onto the pixel of torch.rot90(image0, q) that holds its value: the
    convention of the GPU warp test, on the host."""
    h, w = hw
    img = torch.arange(h * w, dtype=torch.float32).reshape(h, w)
    for q in range(4):
        rot = torch.rot90(img, q, dims=(-2, -1))
        cand = loftr_b200.rotation_candidates(torch.tensor([[w, h]]), torch.tensor([[rot.shape[1], rot.shape[0]]]))
        hq = cand[0, q].double()
        ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64),
                                indexing="ij")
        p = hq @ torch.stack([xs.flatten(), ys.flatten(), torch.ones(h * w, dtype=torch.float64)])
        x1, y1 = p[0] / p[2], p[1] / p[2]
        assert torch.equal(x1, x1.round()) and torch.equal(y1, y1.round()), q
        assert torch.equal(rot[y1.long(), x1.long()], img.flatten()), q


def test_rotation_candidates_reject_bad_arguments():
    s = torch.tensor([[64, 48], [64, 48]])
    cases = [((s[0], s), "size0 must be a real tensor \\[N, 2\\]"), (((64, 48), s), "size0 must be a real tensor"),
             ((s, s.bool()), "size1 must be a real tensor"),
             ((s, s[:1]), "size0 and size1 must have the same N \\(got 2 and 1\\)"),
             ((s, s, torch.ones(2, 2)), "give scale0 and scale1 together"),
             ((s, s, torch.ones(3, 2), torch.ones(3, 2)), "scale0 must be a tensor \\[N, 2\\] with N = 2")]
    for args, match in cases:
        with pytest.raises(ValueError, match="rotation_candidates: " + match):
            loftr_b200.rotation_candidates(*args)


# ------------------------------------------------------------------------------------------------ reference checks
def test_reference_choice_takes_the_largest_count_and_the_smaller_k_on_ties():
    counts = np.array([[3, 7, 7, 1], [0, 0, 0, 0], [5, 5, 5, 5], [0, 0, 0, 9], [2, 1, 0, 0]])
    assert SR.choose(counts).tolist() == [1, 0, 0, 3, 0]
    rs = np.random.RandomState(0)
    rand = rs.randint(0, 4, (200, 6))
    assert np.array_equal(SR.choose(rand), rand.argmax(1))   # numpy's argmax also returns the first maximum


def test_reference_counts_agree_from_flags_and_from_lists():
    rs = np.random.RandomState(1)
    n, k, L = 3, 4, 50
    flags = rs.rand(n * k, L) < rs.uniform(0, 0.5, (n * k, 1))
    flags[4:8] = False   # pair 1: nothing matches under any candidate
    counts = SR.counts_from_flags(flags, k)
    b_ids, i_ids = np.nonzero(flags)   # the list order of the compaction: ascending (c, i)
    assert np.array_equal(SR.counts_from_ids(b_ids, n, k), counts)
    assert SR.choose(counts)[1] == 0 and counts[1].sum() == 0
    lists = {"b_ids": torch.from_numpy(b_ids), "i_ids": torch.from_numpy(i_ids)}
    choice = SR.choose(counts)
    out = SR.winners(lists, choice, k, keys=("b_ids", "i_ids"))
    assert out["b_ids"].tolist() == sorted(out["b_ids"].tolist())
    for b in range(n):
        sel = out["b_ids"] == b
        assert int(sel.sum()) == counts[b, choice[b]]
        assert out["i_ids"][sel].tolist() == np.nonzero(flags[b * k + choice[b]])[0].tolist()
