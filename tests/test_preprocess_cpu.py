"""CPU-side checks of the image front end (`loftr_b200.prepare_images` / `prepare_pairs` / `target_size`): the host
size rule and the float64 reference of the kernel (tests/preprocess_ref.py) against goldens made by the reference's
dataset readers and OpenCV, what is refused before any device work, and the library version guard."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import loftr_b200
import preprocess_ref as ref
import util
from loftr_b200 import _lib, preprocess
from preprocess_cases import GREY_HW, GREY_SEED, IMAGE_CASES, SIZE_CASES, image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_cases.npz"))


@pytest.mark.parametrize("i", range(len(SIZE_CASES)))
def test_target_size_equals_the_reference(i):
    w, h, resize, df = SIZE_CASES[i]
    want = tuple(int(v) for v in GOLD["sizes"][i])
    assert loftr_b200.target_size(w, h, resize, df) == want
    assert ref.target_size(w, h, resize, df) == want


def test_target_size_rounds_ties_to_even_and_truncates():
    ts = loftr_b200.target_size
    assert ts(5, 10, 5, 1) == (2, 5) and ts(7, 10, 5, 1) == (4, 5)   # 2.5 -> 2, 3.5 -> 4
    assert ts(100, 75, 50, 1) == (50, 38)                            # 37.5 -> 38
    assert ts(645, 487) == (640, 480) and ts(645, 487, df=None) == (645, 487)
    assert ts(1296, 968, (640, 480)) == (640, 480) and ts(1296, 968, [643, 485]) == (640, 480)
    assert ts(np.int64(400), np.int32(300), np.int64(832)) == (832, 624)
    assert all(type(v) is int for v in ts(np.int64(400), np.int32(300), np.int64(832)))


@pytest.mark.parametrize("args", [(100, 3, 50), (7, 7, None), (640, 480, (640, 4)), (0, 10, None), (10, -1, None)])
def test_target_size_refuses_a_zero_side(args):
    with pytest.raises(ValueError, match="target_size"):
        loftr_b200.target_size(*args)


@pytest.mark.parametrize("kw", [{"resize": 2.5}, {"resize": True}, {"resize": (640,)}, {"resize": "640"}, {"df": 0},
                                {"df": 2.0}])
def test_target_size_refuses_malformed_options(kw):
    with pytest.raises(ValueError, match="target_size"):
        loftr_b200.target_size(640, 480, **kw)


@pytest.mark.parametrize("name", sorted(IMAGE_CASES))
def test_reference_pipeline_goldens(name):
    """preprocess_ref against read_megadepth_gray / read_scannet_gray: mask and scale exactly, levels within 1.0 of
    cv2.resize's fixed-point result (it rounds to a level; the front end does not), identity size exactly."""
    seed, h, w, resize, df = IMAGE_CASES[name]
    img = image(seed, h, w)
    padded = name.startswith("md_")
    got = ref.prepare([img], resize, df, "square" if padded else None)
    levels = GOLD[name + "_levels"].astype(np.float64)
    assert got["image"].shape == (1, 1, *levels.shape)
    diff = np.abs(got["image"][0, 0] * 255.0 - levels)
    if name.startswith("id_"):
        assert diff.max() == 0.0 and np.array_equal(levels, img)
    else:
        assert diff.max() <= 1.0, diff.max()
        w_new, h_new = got["size"][0]   # the known deviation: after rounding, some valid pixels are one level off
        off = np.abs(np.rint(got["image"][0, 0] * 255.0) - levels)[:h_new, :w_new]
        assert off.max() == 1.0 and 0.05 < off.mean() < 0.2, (off.max(), off.mean())
    if padded:
        assert got["mask"].dtype == bool and np.array_equal(got["mask"][0], GOLD[name + "_mask"])
        assert got["scale"].dtype == np.float32 and np.array_equal(got["scale"][0], GOLD[name + "_scale"])
        w_new, h_new = got["size"][0]
        assert not got["image"][0, 0, h_new:].any() and not got["image"][0, 0, :, w_new:].any()
    else:
        assert got["mask"] is None


def test_grey_equals_opencv():
    rgb = image(GREY_SEED, *GREY_HW, channels=3)
    assert np.array_equal(ref.grey(rgb, "rgb"), GOLD["grey_from_rgb"])
    assert np.array_equal(ref.grey(rgb, "bgr"), GOLD["grey_from_bgr"])
    assert np.array_equal(ref.grey(rgb[..., :1]), rgb[..., 0]) and np.array_equal(ref.grey(rgb[..., 1]), rgb[..., 1])


def _u8(*shape):
    return torch.zeros(shape, dtype=torch.uint8)


REFUSALS = [
    (TypeError, "uint8", dict(images=[torch.zeros(16, 16)])),
    (TypeError, "uint8", dict(images=torch.zeros(2, 16, 16, dtype=torch.int16))),
    (TypeError, "tensor", dict(images=[np.zeros((16, 16), np.uint8)])),
    (TypeError, "list", dict(images="frame.png")),
    (ValueError, r"\[K, h, w\]", dict(images=_u8(16, 16))),
    (ValueError, r"\[K, h, w\]", dict(images=_u8(2, 1, 16, 16, 3))),
    (ValueError, r"\[h, w\]", dict(images=[_u8(2, 16, 16, 3)])),
    (ValueError, "channels", dict(images=[_u8(16, 16, 4)])),
    (ValueError, "channels", dict(images=_u8(2, 16, 16, 2))),
    (ValueError, "no images", dict(images=[])),
    (ValueError, "no images", dict(images=_u8(0, 16, 16))),
    (ValueError, "zero side", dict(images=[_u8(16, 0)])),
    (ValueError, "zero side", dict(images=_u8(2, 0, 16, 3))),
    (ValueError, "target_size", dict(images=[_u8(7, 300)])),
    (ValueError, "same size.*pad_to", dict(images=[_u8(16, 24), _u8(16, 16)])),
    (ValueError, "one square", dict(images=[_u8(16, 24), _u8(16, 16)], pad_to="square")),
    (ValueError, "smaller than an image", dict(images=[_u8(16, 24)], pad_to=(16, 16))),
    (ValueError, "divisible by 8", dict(images=[_u8(16, 24)], pad_to=(20, 24))),
    (ValueError, "divisible by 8", dict(images=[_u8(20, 24)], df=4)),
    (ValueError, "pad_to must be", dict(images=[_u8(16, 24)], pad_to="canvas")),
    (ValueError, "channel_order", dict(images=[_u8(16, 24, 3)], channel_order="gbr")),
    (RuntimeError, "CUDA", dict(images=[_u8(16, 24)], device="cpu")),
]


@pytest.mark.parametrize("exc,match,kw", REFUSALS, ids=[f"{i}-{r[1][:12]}" for i, r in enumerate(REFUSALS)])
def test_refusals_raise_before_any_device_work(monkeypatch, exc, match, kw):
    def no_device(*a, **k):
        raise AssertionError("the refusal must not touch the GPU")

    monkeypatch.setattr(torch.cuda, "current_device", no_device)
    monkeypatch.setattr(_lib.load(), "lb_preprocess_images", no_device, raising=False)
    with pytest.raises(exc, match=match):
        loftr_b200.prepare_images(**kw)
    pair_kw = dict(kw, images0=kw["images"], images1=kw["images"])
    del pair_kw["images"]
    with pytest.raises(exc, match=match):
        loftr_b200.prepare_pairs(**pair_kw)


def test_pairs_refuse_unequal_batches():
    with pytest.raises(ValueError, match="2 images0 but 1 images1"):
        loftr_b200.prepare_pairs(_u8(2, 16, 16), _u8(1, 16, 16))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_images_on_two_devices_are_refused():
    with pytest.raises(ValueError, match="different CUDA devices"):
        loftr_b200.prepare_images([_u8(16, 16).to("cuda:0"), _u8(16, 16).to("cuda:1")])


def test_descs_cache_is_for_device_images():
    with pytest.raises(TypeError, match="descs must be a dict"):
        preprocess._prepare([_u8(16, 16)], [(16, 16)], 16, 16, False, 0, torch.device("cuda:0"), descs=[])
    with pytest.raises(ValueError, match="already be on the device"):
        preprocess._prepare([_u8(16, 16)], [(16, 16)], 16, 16, False, 0, torch.device("cuda:0"), descs={})


def test_front_end_refuses_an_older_library(monkeypatch):
    util.old_library(monkeypatch, 105)
    assert _lib.PREPROCESS_VERSION == 106
    for call in (lambda: loftr_b200.prepare_images([_u8(16, 16)]),
                 lambda: loftr_b200.prepare_pairs([_u8(16, 16)], [_u8(16, 16)])):
        with pytest.raises(RuntimeError, match=r"version 106 or newer.*is version 105"):
            call()
    assert loftr_b200.target_size(640, 480) == (640, 480)   # the host rule needs no library


def test_entry_point_is_bound_and_checks_its_host_arguments():
    lib = _lib.load()
    assert lib.lb_version() >= _lib.PREPROCESS_VERSION
    assert _lib._SINCE["lb_preprocess_images"] == 106
    assert _lib.SIGNATURES["lb_preprocess_images"][1] == lib.lb_preprocess_images.argtypes
    d = (_lib.LbImageDesc * 1)()
    out = C.c_void_p(4096)   # never dereferenced: every call below is refused on its arguments
    for H, W in ((0, 16), (16, -8), (12, 16), (16, 20)):
        assert lib.lb_preprocess_images(d, 1, out, H, W, None, None) != 0
        assert b"divisible by 8" in lib.lb_last_error()
    assert lib.lb_preprocess_images(d, -1, out, 16, 16, None, None) != 0
    assert b"n_images" in lib.lb_last_error()
    assert lib.lb_preprocess_images(None, 1, out, 16, 16, None, None) != 0
    assert b"descs and out are required" in lib.lb_last_error()
    assert lib.lb_preprocess_images(d, 1, None, 16, 16, None, None) != 0
    assert lib.lb_preprocess_images(d, 1, C.c_void_p(4100), 16, 16, None, None) != 0
    assert b"16-byte aligned" in lib.lb_last_error()
    assert lib.lb_preprocess_images(d, 0, out, 16, 16, None, None) == 0   # nothing to do, nothing launched
    assert "preprocess" in [lib.lb_timing_tag_name(i).decode() for i in range(lib.lb_timing_num_tags())]


def test_descriptor_layout_matches_the_header():
    header = open(os.path.join(ROOT, "include", "loftr_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    body = re.search(r"typedef struct LbImageDesc \{(.*?)\} LbImageDesc;", header, re.S).group(1)
    names = [re.findall(r"[A-Za-z_0-9]+", part)[-1] for decl in body.split(";") if decl.strip()
             for part in decl.split(",")]
    assert names == [f[0] for f in _lib.LbImageDesc._fields_]
    assert C.sizeof(_lib.LbImageDesc) == 40 and _lib.LbImageDesc.h.offset == 8 and _lib.LbImageDesc.w_new.offset == 32
