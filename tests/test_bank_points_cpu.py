"""CPU-side checks of `LoFTR.match_points_features` (point queries on bank pairs, DESIGN.md §21): argument validation
and its messages, refusal before anything reaches the matching stages, the binding of its two entries by name and
their argument errors, and the empty pair list / Q = 0."""
import ctypes as C

import pytest
import torch

import loftr_b200
import util
from loftr_b200 import _lib

WHO = "match_points_features"


def _model():
    return loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).eval()


def _idx(*v):
    return torch.tensor(v, dtype=torch.int64)


@pytest.fixture
def no_stages(monkeypatch):
    return util.stages_unreachable(monkeypatch, _model())


def _call(model, bank0=None, idx0=None, bank1=None, idx1=None, pts=None, **kw):
    bank0 = util.host_bank(model) if bank0 is None else bank0
    bank1 = bank0 if bank1 is None else bank1
    idx0 = _idx(0, 1) if idx0 is None else idx0
    idx1 = _idx(1, 2) if idx1 is None else idx1
    pts = torch.zeros(idx0.shape[0] if torch.is_tensor(idx0) else 2, 4, 2) if pts is None else pts
    return model.match_points_features(bank0, idx0, bank1, idx1, pts, **kw)


# ------------------------------------------------------------------------------------------------ bank arguments
def test_bank_checks_name_the_call(no_stages):
    m = no_stages
    bank = util.host_bank(m)
    with pytest.raises(TypeError, match=rf"{WHO}: `feats0` must be the ImageFeatures of extract_features"):
        _call(m, bank0=object(), bank1=bank)
    with pytest.raises(TypeError, match=rf"{WHO}: `idx1` must be an int32 or int64 tensor \(got torch.float32\)"):
        _call(m, idx1=torch.zeros(2))
    with pytest.raises(TypeError, match=rf"{WHO}: `idx0` must be an int32 or int64 tensor \(got list\)"):
        _call(m, idx0=[0, 1], pts=torch.zeros(2, 4, 2))
    with pytest.raises(ValueError, match=rf"{WHO}: `idx0` is on meta, the model on cpu"):
        _call(m, idx0=_idx(0, 1).to("meta"))
    with pytest.raises(ValueError, match=rf"{WHO}: `idx1` must be one-dimensional \(got shape \(2, 1\)\)"):
        _call(m, idx1=_idx(0, 1)[:, None])
    with pytest.raises(IndexError, match=rf"{WHO}: `idx1` holds indices in \[1, 3\], outside the bank's \[0, 3\)"):
        _call(m, idx1=_idx(1, 3))
    with pytest.raises(IndexError, match=rf"{WHO}: `idx0` holds indices in \[-1, 0\]"):
        _call(m, idx0=_idx(-1, 0))
    with pytest.raises(ValueError, match=rf"{WHO}: idx0 and idx1 must have the same length \(2 vs 1\)"):
        _call(m, idx1=_idx(1))
    with pytest.raises(ValueError, match=rf"{WHO}: either both banks carry masks or neither"):
        _call(m, bank0=util.host_bank(m, masks=True), bank1=bank)
    with pytest.raises(ValueError, match=rf"{WHO}: give scale0 and scale1 together"):
        _call(m, scale0=torch.ones(3, 2))


def test_a_bank_tied_to_other_weights_raises(no_stages):
    m = no_stages
    bank = util.host_bank(m)
    with torch.no_grad():
        m.backbone.conv1.weight.add_(0.0)   # an in-place update: a new _version
    with pytest.raises(RuntimeError, match=rf"{WHO}: `feats0` was extracted with other backbone weights"):
        _call(m, bank0=bank)


# ------------------------------------------------------------------------------------------------ query arguments
@pytest.mark.parametrize("points, err, msg", [
    (torch.zeros(2, 4, 2, dtype=torch.float64), TypeError, "points0 must be a float32 tensor"),
    ("not a tensor", TypeError, r"points0 must be a float32 tensor \(got str\)"),
    (torch.zeros(2, 4), ValueError, r"points0 must be \[N, Q, 2\] with N = 2 pairs"),
    (torch.zeros(3, 4, 2), ValueError, r"points0 must be \[N, Q, 2\] with N = 2 pairs \(got \(3, 4, 2\)\)"),
    (torch.zeros(2, 4, 3), ValueError, r"points0 must be \[N, Q, 2\]"),
])
def test_points_are_checked_against_the_pair_list(no_stages, points, err, msg):
    with pytest.raises(err, match=f"{WHO}: {msg}"):
        _call(no_stages, pts=points)


def test_valid0_devices_and_the_guide_are_checked(no_stages):
    m = no_stages
    with pytest.raises(TypeError, match=f"{WHO}: valid0 must be a bool tensor"):
        _call(m, valid0=torch.ones(2, 4, dtype=torch.uint8))
    with pytest.raises(ValueError, match=rf"{WHO}: valid0 must be \[N, Q\] = \(2, 4\) \(got \(2, 5\)\)"):
        _call(m, valid0=torch.ones(2, 5, dtype=torch.bool))
    # well-formed host arguments: the device check stops them, Q = 0 and an empty pair list included
    for idx, q in ((_idx(0, 1), 4), (_idx(0, 1), 0), (_idx(), 4)):
        with pytest.raises(ValueError, match=f"{WHO}: `points0` must be a CUDA tensor"):
            _call(m, idx0=idx, idx1=idx, pts=torch.zeros(idx.numel(), q, 2))


def test_guide_and_scale_errors_come_before_any_gather(monkeypatch):
    """With the queries on the model's device (here: a host model given host points that pass), the guide and the
    scale shapes are still checked before anything is gathered or matched."""
    m = _model()
    from loftr_b200 import loftr as LM
    monkeypatch.setattr(LM, "_check_devices", lambda *a, **k: None)
    for name in ("_match_points", "_coarse_tokens", "_backbone"):
        monkeypatch.setattr(m, name, lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached")))
    with pytest.raises(ValueError, match=rf"{WHO}: guide\['model'\] must be \[N, 3, 3\] with N = 2 pairs"):
        _call(m, guide={"kind": "homography", "model": torch.eye(3)[None], "radius": 8.0})
    with pytest.raises(ValueError, match=rf"{WHO}: guide\['radius'\] must be finite and positive"):
        _call(m, guide={"kind": "homography", "model": torch.eye(3).repeat(2, 1, 1), "radius": float("inf")})
    with pytest.raises(TypeError, match=f"{WHO}: guide must be a dict"):
        _call(m, guide=[1])
    with pytest.raises(ValueError, match=rf"{WHO}: scale1 must be \[3, 2\] \(got \(2, 2\)\)"):
        _call(m, scale0=torch.ones(3, 2), scale1=torch.ones(2, 2))
    for idx, q in ((_idx(0, 1), 0), (_idx(), 4)):   # also for empty outputs
        with pytest.raises(ValueError, match=rf"{WHO}: scale0 must be \[3, 2\]"):
            _call(m, idx0=idx, idx1=idx, pts=torch.zeros(idx.numel(), q, 2), scale0=torch.ones(1, 2),
                  scale1=torch.ones(3, 2))


def test_empty_pair_list_and_q0_give_empty_outputs(monkeypatch):
    m = _model()
    from loftr_b200 import loftr as LM
    monkeypatch.setattr(LM, "_check_devices", lambda *a, **k: None)
    for name in ("_match_points", "_coarse_tokens", "_backbone"):
        monkeypatch.setattr(m, name, lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached")))
    bank = util.host_bank(m, masks=True)
    for idx, q in ((_idx(0, 2), 0), (_idx(), 5)):
        mine = {"kept": 1}
        out = m.match_points_features(bank, idx, bank, idx, torch.zeros(idx.numel(), q, 2), data=mine,
                                      scale0=torch.ones(3, 2), scale1=torch.ones(3, 2))
        assert out is mine and out["kept"] == 1
        assert out["bs"] == idx.numel() and out["hw0_i"] == (96, 128) and out["hw1_f"] == (48, 64)
        for k, (dtype, d) in LM._QUERY_KEYS.items():
            assert out[k].dtype == dtype and tuple(out[k].shape) == (idx.numel(), q) + ((d,) if d else ()), k
        assert not {"mask0", "mask1", "scale0", "scale1", "guide"} & set(out)


def test_match_points_still_refuses_a_guide():
    m = _model()
    guide = {"kind": "homography", "model": torch.eye(3)[None], "radius": 8.0}
    with pytest.raises(ValueError, match=r"match_points: data\['guide'\] is not supported"):
        m.match_points({"image0": torch.zeros(1, 1, 8, 8), "image1": torch.zeros(1, 1, 8, 8), "guide": guide},
                       torch.zeros(1, 4, 2))


# ------------------------------------------------------------------------------------------------ binding by name
def test_entries_are_bound_only_where_exported(monkeypatch):
    lib = _lib.load()
    assert _lib.BANK_POINTS_ENTRIES == ("lb_coarse_query_guided", "lb_fine_preprocess_centres_indexed")
    for name in _lib.BANK_POINTS_ENTRIES:
        assert name not in _lib._SINCE and name in _lib._OPTIONAL
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    assert lib.lb_version() == 110
    _lib.require_entries(_lib.BANK_POINTS_ENTRIES, WHO)
    old = util.load_without(monkeypatch, _lib.BANK_POINTS_ENTRIES)
    assert not any(hasattr(old, n) for n in _lib.BANK_POINTS_ENTRIES)
    assert old.lb_coarse_query.argtypes == _lib.SIGNATURES["lb_coarse_query"][1]   # the rest still binds
    _lib.require_entries(_lib.POINTS_ENTRIES + _lib.GUIDE_ENTRIES + _lib.SEARCH_ENTRIES, "other paths")
    m = _model()
    bank = util.host_bank(m)
    with pytest.raises(RuntimeError, match=rf"{WHO} needs lb_coarse_query_guided, which .* \(version 110\) does not "
                                           "export"):
        _call(m, bank0=bank)


def test_coarse_query_guided_checks_its_arguments():
    lib = _lib.load()
    a, q = _lib.LbCoarseMatchArgs(), _lib.LbCoarseQueryArgs()
    model = torch.zeros(9)
    g = lambda kind=0, ptr=model.data_ptr(), radius=4.0: C.byref(_lib.LbCoarseGuide(kind, ptr, radius))
    cases = [(None, 2, b"the guide model is null"),
             (g(ptr=None), 2, b"the guide model is null"),
             (g(kind=2), 2, b"unknown guide kind 2"),
             (g(radius=0.0), 2, b"the radius must be finite and positive (got 0)"),
             (g(radius=-1.0), 2, b"the radius must be finite and positive (got -1)"),
             (g(radius=float("nan")), 2, b"the radius must be finite and positive (got nan)"),
             (g(radius=float("inf")), 1, b"the radius must be finite and positive (got inf)"),
             (g(), 3, b"operand_planes must be 1 (fp16) or 2 (split) (got 3)"),
             (g(), 0, b"operand_planes must be 1 (fp16) or 2 (split) (got 0)")]
    for guide, planes, msg in cases:
        assert lib.lb_coarse_query_guided(C.byref(a), C.byref(q), guide, planes, None, 0, None) != 0
        err = lib.lb_last_error()
        assert msg in err and err.startswith(b"lb_coarse_query_guided: "), (msg, err)
    # a good guide and Q = 0: nothing to do
    assert lib.lb_coarse_query_guided(C.byref(a), C.byref(q), g(), 2, None, 0, None) == 0
    # the guided match entry keeps its messages
    assert lib.lb_coarse_match_guided(C.byref(a), g(kind=5), 0, 0, None, 0, None) != 0
    assert lib.lb_last_error() == b"lb_coarse_match_guided: unknown guide kind 5"


def test_fine_preprocess_centres_indexed_checks_its_arguments():
    lib = _lib.load()
    buf = torch.zeros(16, dtype=torch.int32)
    p = buf.data_ptr()
    f = _lib.LbFinePreprocessArgs()
    f.M = 4
    for args in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        assert lib.lb_fine_preprocess_centres_indexed(C.byref(f), *args, None, 0, None) != 0
        assert lib.lb_last_error() == (b"lb_fine_preprocess_centres_indexed: centres, inside, img_idx0 and img_idx1 "
                                       b"are required")
    f.M_live = p
    assert lib.lb_fine_preprocess_centres_indexed(C.byref(f), p, p, p, p, None, 0, None) != 0
    assert b"lb_fine_preprocess_centres_indexed: M_live is not supported" in lib.lb_last_error()
    f.M, f.M_live = 0, None   # M = 0: nothing to do, NULL tables allowed
    assert lib.lb_fine_preprocess_centres_indexed(C.byref(f), None, None, None, None, None, 0, None) == 0
