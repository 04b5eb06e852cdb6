"""CPU-side checks of image1-side point queries and round trips (DESIGN.md §22): argument validation and its messages
for `match_points` and `match_points_features`, refusal before any matching stage, the binding of the two entries by
name, their argument errors (a workspace too small for the query-only entry among them), and Q = 0 / an empty pair
list, which launch nothing."""
import ctypes as C

import pytest
import torch

import loftr_b200
import util
from loftr_b200 import _lib
from loftr_b200 import loftr as LM


def _model():
    return loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).eval()


def _idx(*v):
    return torch.tensor(v, dtype=torch.int64)


def _data():
    return {"image0": torch.zeros(2, 1, 96, 128), "image1": torch.zeros(2, 1, 96, 128)}


@pytest.fixture
def no_stages(monkeypatch):
    return util.stages_unreachable(monkeypatch, _model())


def _calls(m):
    """(who, call(**query kwargs)) for both query methods on two pairs."""
    bank = util.host_bank(m)
    return [("match_points", lambda **kw: m.match_points(_data(), **kw)),
            ("match_points_features", lambda **kw: m.match_points_features(bank, _idx(0, 1), bank, _idx(1, 2), **kw))]


# ------------------------------------------------------------------------------------------------ validation
def test_one_image_of_queries_and_a_bool_round_trip(no_stages):
    pts = torch.zeros(2, 4, 2)
    ok = torch.ones(2, 4, dtype=torch.bool)
    for who, call in _calls(no_stages):
        with pytest.raises(ValueError, match=rf"{who}: give the queries of one image: points0 \(and valid0\) or "
                                             r"points1 \(and valid1\)"):
            call(points0=pts, points1=pts)
        with pytest.raises(ValueError, match=f"{who}: give the queries of one image"):
            call(valid0=ok, points1=pts)
        with pytest.raises(ValueError, match=f"{who}: valid1 is given without points1"):
            call(points0=pts, valid1=ok)
        for bad in (1, None, "yes", torch.tensor(True)):
            with pytest.raises(TypeError, match=f"{who}: round_trip must be a bool"):
                call(points1=pts, round_trip=bad)
        # neither: the points0 check of a call without points1, as before
        with pytest.raises(TypeError, match=rf"{who}: points0 must be a float32 tensor \(got NoneType\)"):
            call()


@pytest.mark.parametrize("points, err, msg", [
    (torch.zeros(2, 4, 2, dtype=torch.float64), TypeError, "points1 must be a float32 tensor"),
    ("not a tensor", TypeError, r"points1 must be a float32 tensor \(got str\)"),
    (torch.zeros(2, 4), ValueError, r"points1 must be \[N, Q, 2\] with N = 2 pairs"),
    (torch.zeros(3, 4, 2), ValueError, r"points1 must be \[N, Q, 2\] with N = 2 pairs \(got \(3, 4, 2\)\)"),
])
def test_points1_shapes_and_dtypes(no_stages, points, err, msg):
    for who, call in _calls(no_stages):
        for rt in (False, True):
            with pytest.raises(err, match=f"{who}: {msg}"):
                call(points1=points, round_trip=rt)


def test_valid1_and_devices(no_stages):
    pts = torch.zeros(2, 4, 2)
    for who, call in _calls(no_stages):
        with pytest.raises(TypeError, match=f"{who}: valid1 must be a bool tensor"):
            call(points1=pts, valid1=torch.ones(2, 4, dtype=torch.uint8))
        with pytest.raises(ValueError, match=rf"{who}: valid1 must be \[N, Q\] = \(2, 4\) \(got \(2, 5\)\)"):
            call(points1=pts, valid1=torch.ones(2, 5, dtype=torch.bool))
        # well-formed host arguments: the device check stops them, Q = 0 included
        for q in (4, 0):
            with pytest.raises(ValueError, match=f"{who}: `(image0|points1)` must be a CUDA tensor"):
                call(points1=torch.zeros(2, q, 2), round_trip=True)
        with pytest.raises(ValueError, match=f"{who}: `(image0|points0)` must be a CUDA tensor"):
            call(points0=pts, round_trip=True)


def test_rectified_calls_refuse_image1_queries_and_round_trips(monkeypatch, no_stages):
    monkeypatch.setattr(LM, "_check_devices", lambda *a, **k: None)
    m = no_stages
    monkeypatch.setattr(m, "_rectified", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached")))
    data = dict(_data(), rectify1=torch.eye(3).repeat(2, 1, 1))
    for kw in ({"points1": torch.zeros(2, 4, 2)}, {"points0": torch.zeros(2, 4, 2), "round_trip": True}):
        with pytest.raises(ValueError, match=r"match_points: points1 and round_trip cannot be combined with "
                                             r"data\['rectify1'\]"):
            m.match_points(data, **kw)


def test_q0_and_an_empty_pair_list_give_empty_outputs(monkeypatch):
    m = _model()
    monkeypatch.setattr(LM, "_check_devices", lambda *a, **k: None)
    for name in ("_coarse_tokens", "_backbone", "_backbone_pairs"):
        monkeypatch.setattr(m, name, lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached")))
    launches = _lib.load().lb_launch_count
    n_launch = launches()
    bank = util.host_bank(m)
    side1 = {"qpts1_f", "qpts0_c", "qpts0_f", "qexpec_f", "qconf", "q_i_ids", "q_j_ids", "qmutual", "qvalid",
             "qinside"}
    back = {"qback_pts", "qback_conf", "qback_valid", "qback_inside", "qfb_err"}
    for rt in (False, True):
        for idx, q in ((_idx(0, 2), 0), (_idx(), 5)):
            out = m.match_points_features(bank, idx, bank, idx, points1=torch.zeros(idx.numel(), q, 2), round_trip=rt)
            keys = side1 | (back if rt else set())
            assert keys <= set(out) and "qpts1_c" not in out and (back <= set(out)) == rt
            for k in keys:
                d = {"qpts1_f": 2, "qpts0_c": 2, "qpts0_f": 2, "qback_pts": 2, "qexpec_f": 3}.get(k)
                assert tuple(out[k].shape) == (idx.numel(), q) + ((d,) if d else ()), k
        data = _data()
        m.match_points(data, points0=torch.zeros(2, 0, 2), round_trip=rt)
        assert {"qpts0_f", "qpts1_c", "qpts1_f"} <= set(data) and (back <= set(data)) == rt
        if rt:
            assert data["qback_pts"].shape == (2, 0, 2) and data["qfb_err"].dtype == torch.float32
    assert launches() == n_launch


# ------------------------------------------------------------------------------------------------ binding by name
def test_entries_are_bound_only_where_exported(monkeypatch):
    lib = _lib.load()
    assert _lib.SIDE_POINTS_ENTRIES == ("lb_coarse_query_side", "lb_coarse_query_reuse")
    for name in _lib.SIDE_POINTS_ENTRIES:
        assert name not in _lib._SINCE and name in _lib._OPTIONAL
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    assert lib.lb_version() == 110
    old = util.load_without(monkeypatch, _lib.SIDE_POINTS_ENTRIES)
    assert not any(hasattr(old, n) for n in _lib.SIDE_POINTS_ENTRIES)
    _lib.require_entries(_lib.POINTS_ENTRIES + _lib.BANK_POINTS_ENTRIES, "the image0 queries")
    m = _model()
    pts = torch.zeros(2, 4, 2)
    for who, call in _calls(m):
        for kw in ({"points1": pts}, {"points0": pts, "round_trip": True}):
            with pytest.raises(RuntimeError, match=rf"{who} needs lb_coarse_query_side, which .* \(version 110\) does "
                                                   "not export"):
                call(**kw)
        with pytest.raises(ValueError, match=f"{who}: `(image0|points0)` must be a CUDA tensor"):   # image0 queries run
            call(points0=pts)


# ------------------------------------------------------------------------------------------------ C entries
def _query_args(q=4):
    pts = torch.zeros(8, dtype=torch.float32)
    qa = _lib.LbCoarseQueryArgs()
    qa.Q, qa.points0 = q, pts.data_ptr()
    qa.H0, qa.W0, qa.Hf0, qa.Wf0, qa.stride, qa.fine_scale = 96, 128, 48, 64, 4, 2.0
    a = _lib.LbCoarseMatchArgs()
    a.n_pairs, a.L, a.S, a.h0c, a.w0c, a.h1c, a.w1c = 2, 192, 192, 12, 16, 12, 16
    return a, qa, pts


def test_coarse_query_side_checks_its_arguments():
    lib = _lib.load()
    a, q, keep = _query_args()
    model = torch.zeros(9)
    g = lambda kind=0, radius=4.0: C.byref(_lib.LbCoarseGuide(kind, model.data_ptr(), radius))
    cases = [(None, 2, 2, b"side must be 0 (image0) or 1 (image1) (got 2)"),
             (None, -1, 2, b"side must be 0 (image0) or 1 (image1) (got -1)"),
             (None, 1, 3, b"operand_planes must be 1 (fp16) or 2 (split) (got 3)"),
             (g(kind=2), 1, 2, b"unknown guide kind 2"),
             (g(radius=float("nan")), 0, 1, b"the radius must be finite and positive (got nan)"),
             (C.byref(_lib.LbCoarseGuide(0, None, 4.0)), 1, 2, b"the guide model is null")]
    for guide, side, planes, msg in cases:
        assert lib.lb_coarse_query_side(C.byref(a), C.byref(q), guide, side, planes, None, 0, None) != 0
        err = lib.lb_last_error()
        assert msg in err and err.startswith(b"lb_coarse_query_side: "), (msg, err)
    q.Q = 0   # nothing to do, with or without a guide
    for guide in (None, g()):
        assert lib.lb_coarse_query_side(C.byref(a), C.byref(q), guide, 1, 2, None, 0, None) == 0


def test_coarse_query_reuse_checks_its_arguments_and_the_workspace_size():
    lib = _lib.load()
    need = lib.lb_coarse_match_workspace_bytes(2, 192, 192)
    ws = torch.zeros(need, dtype=torch.uint8)

    def err(mutate, ws_ptr=ws.data_ptr(), nbytes=need, side=1):
        a, q, keep = _query_args()
        mutate(a, q)
        assert lib.lb_coarse_query_reuse(C.byref(a), C.byref(q), side, ws_ptr, nbytes, None) != 0
        msg = lib.lb_last_error()
        assert msg.startswith(b"lb_coarse_query_reuse: "), msg
        return msg.decode()

    none = lambda a, q: None
    assert "side must be 0 (image0) or 1 (image1) (got 3)" in err(none, side=3)
    assert err(lambda a, q: setattr(q, "points0", None)).endswith("points0 is null")
    assert "bad fine grid (stride 0" in err(lambda a, q: setattr(q, "stride", 0))
    assert err(lambda a, q: setattr(a, "L", 191)).endswith("L/S do not match the coarse grid sizes")
    assert err(lambda a, q: setattr(a, "match_type", 7)).endswith("unknown match_type 7")
    assert err(none, ws_ptr=None).endswith("workspace pointer is null")
    assert err(none, nbytes=need - 257).endswith(f"workspace of {need - 257} bytes is too small for 2 pairs of "
                                                 f"192 x 192 cells (need {need})")
    # a workspace sized for fewer pairs is refused as well
    small = lib.lb_coarse_match_workspace_bytes(1, 192, 192)
    assert "is too small" in err(none, nbytes=small)
    for q_, n in ((0, 2), (4, 0)):   # nothing to do: no launch, no check of the rest
        a, q, keep = _query_args(q_)
        a.n_pairs = n
        assert lib.lb_coarse_query_reuse(C.byref(a), C.byref(q), 0, None, 0, None) == 0
