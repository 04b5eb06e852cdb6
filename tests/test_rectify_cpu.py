"""CPU-side checks of rectified matching (data["rectify1"], DESIGN.md §19): the shared validator and the callers that
refuse rectify1, the binding of lb_rectify_images / lb_rectify_points by name and their argument errors, and
self-checks of the float64 references (tests/rectify_ref.py)."""
import numpy as np
import pytest
import torch

import loftr_b200
import rectify_ref as RR
import util
from loftr_b200 import _lib
from loftr_b200.loftr import CapturedMatcher, check_rectify


def _eye(n=2, **kw):
    return torch.eye(3, **kw).repeat(n, 1, 1)


@pytest.mark.parametrize("model, exc, match", [
    (np.eye(3, dtype=np.float32)[None].repeat(2, 0), TypeError, "rectify1 must be a float32 tensor"),
    (_eye(dtype=torch.float64), TypeError, "rectify1 must be a float32 tensor"),
    (_eye(3), ValueError, r"rectify1 must be \[N, 3, 3\] with N = 2"),
    (torch.zeros(2, 9), ValueError, r"rectify1 must be \[N, 3, 3\]"),
    (_eye(device="meta"), ValueError, "rectify1 is on meta, the images on cpu"),
    (_eye(), ValueError, "rectify1 must be a CUDA tensor"),
], ids=["numpy", "f64", "n", "shape", "device", "host"])
def test_validator_rejects(model, exc, match):
    with pytest.raises(exc, match="forward: " + match):
        check_rectify(model, 2, torch.device("cpu"), "forward")


def _model():
    return loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).eval()


def test_callers_refuse_rectify1_with_a_guide_and_in_a_captured_matcher():
    m = _model()
    guide = {"kind": "homography", "model": _eye(1), "radius": 8.0}
    data = {"image0": torch.zeros(1, 1, 8, 8), "image1": torch.zeros(1, 1, 8, 8), "rectify1": _eye(1), "guide": guide}
    with pytest.raises(ValueError, match=r"forward_static: data\['rectify1'\] cannot be combined with data\['guide'\]"):
        m._rectified(data, "forward_static")
    cap = CapturedMatcher.__new__(CapturedMatcher)   # refused before the graph or the weights are read
    cap.graph = None
    with pytest.raises(ValueError, match=r"CapturedMatcher: data\['rectify1'\] is not supported"):
        cap({"image0": torch.zeros(1, 1, 8, 8), "rectify1": _eye(1)})


def test_rectified_input_is_validated_before_any_launch():
    m = _model()
    base = {"image0": torch.zeros(2, 1, 16, 16), "image1": torch.zeros(2, 1, 24, 32)}
    for extra, match in (({"rectify1": _eye(3)}, r"rectify1 must be \[N, 3, 3\] with N = 2"),
                         ({"rectify1": _eye()}, "rectify1 must be a CUDA tensor")):
        with pytest.raises(ValueError, match="forward: " + match):
            m._rectified(dict(base, **extra), "forward")


def test_warp_images_rejects_bad_arguments():
    img = torch.zeros(2, 1, 24, 32)
    cases = [((torch.zeros(2, 24, 32), _eye(), (16, 16)), ValueError, r"images1 must be a float32 tensor \[N, 1"),
             ((img.double(), _eye(), (16, 16)), ValueError, "images1 must be a float32 tensor"),
             ((img, _eye(), (16, 12)), ValueError, r"hw must be \(H, W\), positive multiples of 8"),
             ((img, _eye(), (0, 16)), ValueError, "hw must be"),
             ((img, _eye(), 16), ValueError, "hw must be"),
             ((img, _eye(), (16, 16), torch.ones(2, 2)), ValueError, "give scale0 and scale1 together"),
             ((img, _eye(), (16, 16), torch.ones(3, 2), torch.ones(3, 2)), ValueError,
              r"scale0 must be a tensor \[N, 2\]"),
             ((img, _eye(3), (16, 16)), ValueError, r"warp_images: rectify1 must be \[N, 3, 3\] with N = 2"),
             ((img, _eye(), (16, 16)), ValueError, "warp_images: rectify1 must be a CUDA tensor")]
    for args, exc, match in cases:
        with pytest.raises(exc, match=match):
            loftr_b200.warp_images(*args)


def test_rectify_entries_are_bound_only_where_exported(monkeypatch):
    """lb_rectify_images / lb_rectify_points come without a version step, found by name like the guided and point
    entries: the shipped build exports and binds them; a build without them still loads, and only rectify1 is
    refused."""
    lib = _lib.load()
    assert _lib.RECTIFY_ENTRIES == ("lb_rectify_images", "lb_rectify_points")
    for name in _lib.RECTIFY_ENTRIES:
        assert name not in _lib._SINCE and name in _lib._OPTIONAL
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    assert lib.lb_version() == 110
    _lib.require_entries(_lib.RECTIFY_ENTRIES, "rectified matching")
    names = {lib.lb_timing_tag_name(i).decode() for i in range(lib.lb_timing_num_tags())}
    assert "rectify" in names
    old = util.load_without(monkeypatch, _lib.RECTIFY_ENTRIES)
    assert not hasattr(old, "lb_rectify_images") and not hasattr(old, "lb_rectify_points")
    assert old.lb_coarse_match_guided.argtypes == _lib.SIGNATURES["lb_coarse_match_guided"][1]   # the rest still binds
    _lib.require_entries(_lib.GUIDE_ENTRIES + _lib.POINTS_ENTRIES, "other paths")
    with pytest.raises(RuntimeError, match=r"forward: rectified matching needs lb_rectify_images.*\(version 110\)"):
        check_rectify(_eye(), 2, torch.device("cpu"), "forward")


def test_rectify_entries_check_their_arguments():
    lib = _lib.load()
    buf = torch.zeros(64)
    p = buf.data_ptr()
    img_cases = [((p, 1, 8, 8, p, None, None, p, 12, 16), b"canvas 12x16 must be positive and divisible by 8"),
                 ((p, 1, 8, 8, p, None, None, p, 0, 16), b"canvas 0x16 must be positive"),
                 ((p, -1, 8, 8, p, None, None, p, 8, 8), b"n=-1 must be in [0, 65535]"),
                 ((p, 65536, 8, 8, p, None, None, p, 8, 8), b"n=65536 must be in [0, 65535]"),
                 ((p, 1, 0, 8, p, None, None, p, 8, 8), b"image1 size 0x8 must be positive"),
                 ((None, 1, 8, 8, p, None, None, p, 8, 8), b"image1, models and out are required"),
                 ((p, 1, 8, 8, None, None, None, p, 8, 8), b"image1, models and out are required"),
                 ((p, 1, 8, 8, p, None, None, None, 8, 8), b"image1, models and out are required"),
                 ((p, 1, 8, 8, p, None, None, p + 4, 8, 8), b"out is not 16-byte aligned")]
    for args, msg in img_cases:
        assert lib.lb_rectify_images(*args, None) != 0
        assert msg in lib.lb_last_error(), (args, lib.lb_last_error())
    assert lib.lb_rectify_images(p, 0, 8, 8, p, None, None, p, 8, 8, None) == 0   # nothing to do: no device needed
    pt_cases = [((p, p, -1, None, p, 1, None, None, 8, 8, 8, 8, None, 1, p, None), b"m=-1 and n_pairs=1"),
                ((p, p, 4, None, p, -1, None, None, 8, 8, 8, 8, None, 1, p, None), b"must not be negative"),
                ((p, p, 4, None, p, 1, None, None, 8, 0, 8, 8, None, 1, p, None), b"image sizes 8x0 and 8x8"),
                ((p, p, 4, None, p, 1, None, None, 8, 8, 12, 8, p, 1, p, None), b"mask1 needs image1 sides divisible"),
                ((p, p, 4, None, p, 1, None, None, 8, 8, 8, 16, p, 1, p, None), b"w1c = W1 / 8 (got 8x16, w1c=1)"),
                ((None, p, 4, None, p, 1, None, None, 8, 8, 8, 8, None, 1, p, None), b"pts, pair_ids, models and out"),
                ((p, None, 4, None, p, 1, None, None, 8, 8, 8, 8, None, 1, p, None), b"pts, pair_ids, models and out"),
                ((p, p, 4, None, None, 1, None, None, 8, 8, 8, 8, None, 1, p, None), b"pts, pair_ids, models and out"),
                ((p, p, 4, None, p, 1, None, None, 8, 8, 8, 8, None, 1, None, None), b"pts, pair_ids, models and out")]
    for args, msg in pt_cases:
        assert lib.lb_rectify_points(*args, None) != 0
        assert msg in lib.lb_last_error(), (args, lib.lb_last_error())
    assert lib.lb_rectify_points(None, None, 0, None, None, 0, None, None, 8, 8, 8, 8, None, 1, None, None, None) == 0


# ------------------------------------------------------------------------------------------------ oracle self-checks
def _images(n=2, h=24, w=40, seed=0):
    return torch.from_numpy(np.random.RandomState(seed).rand(n, 1, h, w).astype(np.float32))


def test_oracle_identity_is_an_exact_copy_and_nan_models_are_the_identity():
    img = _images()
    scale = torch.tensor([[1.5, 2.0], [0.75, 1.25]])
    for models in (torch.eye(3).repeat(2, 1, 1), torch.full((2, 3, 3), float("nan")), -torch.eye(3).repeat(2, 1, 1)):
        for s in (None, scale):
            out, u, v = RR.warp(img, models, (24, 40), s, s)
            assert torch.allclose(out, img.double(), rtol=0, atol=1e-12)
            assert torch.equal(u[0], torch.arange(40, dtype=torch.float64).expand(24, 40))


def test_oracle_integer_translation_is_an_exact_shift():
    img = _images()
    tx, ty = 5, -3
    H = torch.tensor([[1.0, 0, tx], [0, 1, ty], [0, 0, 1]]).repeat(2, 1, 1)
    out, _, _ = RR.warp(img, H, (32, 48))
    want = torch.zeros(2, 1, 32, 48, dtype=torch.float64)
    want[:, :, 3:24 + 3, :40 - tx] = img.double()[:, :, :, tx:]   # out[y, x] = img[y + ty, x + tx]
    assert torch.allclose(out, want, rtol=0, atol=1e-12)


def test_oracle_half_turn_about_the_centre_is_an_exact_flip():
    img = _images(h=24, w=32)
    H = torch.tensor([[-1.0, 0, 31], [0, -1, 23], [0, 0, 1]]).repeat(2, 1, 1)
    out, _, _ = RR.warp(img, H, (24, 32))
    assert torch.allclose(out, img.double().flip(-1, -2), rtol=0, atol=1e-12)
    out_neg, _, _ = RR.warp(img, -H, (24, 32))   # -H is the same homography
    assert torch.equal(out_neg, out)


def test_oracle_horizon_and_back_mapping_round_trip():
    rs = np.random.RandomState(4)
    n, hw0, hw1 = 3, (48, 64), (40, 56)
    s0 = torch.from_numpy(rs.uniform(0.8, 1.5, (n, 2)))
    s1 = torch.from_numpy(rs.uniform(0.8, 1.5, (n, 2)))
    Hs = torch.from_numpy(np.stack([np.eye(3) + rs.normal(0, 0.05, (3, 3)) * [[1, 1, 20], [1, 1, 20], [1e-3, 1e-3, 0]]
                                    for _ in range(n)]))
    pts = torch.from_numpy(rs.uniform(0, 60, (200, 2)))
    ids = torch.from_numpy(rs.randint(0, n, 200))
    x1, inside = RR.map_back(pts, ids, Hs, hw0, hw1, s0, s1)
    assert inside.any() and (~inside).any()
    back, _ = RR.map_back(x1, ids, torch.linalg.inv(Hs), hw1, hw0, s1, s0)
    assert torch.allclose(back, pts, rtol=0, atol=1e-9)
    # a model whose horizon crosses the canvas: w <= 0 samples 0 and maps to NaN, not inside
    Hh = torch.tensor([[1.0, 0, 0], [0, 1, 0], [-0.05, 0, 1.6]]).repeat(n, 1, 1)   # w = 0 at x = 32 (centre w > 0)
    out, u, _ = RR.warp(_images(n, 48, 64), Hh, hw0)
    assert torch.isnan(u[:, :, 33:]).all() and (out[:, 0, :, 33:] == 0).all() and torch.isfinite(u[:, :, :32]).all()
    x1, inside = RR.map_back(torch.tensor([[40.0, 5.0], [10.0, 5.0]]), [0, 0], Hh, hw0, hw1)
    assert torch.isnan(x1[0]).all() and not inside[0] and inside[1]
    mask = torch.zeros(n, 5, 7, dtype=torch.bool)
    _, inside_m = RR.map_back(torch.tensor([[10.0, 5.0]]), [0], Hh, hw0, hw1, mask1=mask)
    assert not inside_m[0]
