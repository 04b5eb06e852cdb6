"""The fp16 backbone (`backbone_impl="b200_fp16"`, lb_backbone_forward_fp16) on the GPU.

Per output map, the error against the float64 module is held to twice the error of the float64 emulation of the same
semantics (tests/backbone_ref.py) plus 1e-6 of the map's scale: the kernels' fp32 accumulation order is the
only difference from the emulation.  Bits do not depend on the workspace's padding, on repetition or on the batch, and
the whole matcher runs unchanged on top of the new backbone."""
import copy

import numpy as np
import pytest
import torch

import backbone_ref as B
import loftr_b200
import util
from cases import BASELINE_CASES, CASES, build_inputs
from match_cap_ref import LIST_KEYS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_CASE = {c["name"]: c for c in CASES}


def _tc(model):
    from loftr_b200.loftr import TensorCoreBackbone
    return TensorCoreBackbone(model.backbone, precision="fp16")


@pytest.mark.parametrize("shape", [(1, 16, 16), (16, 136, 200), (1, 88, 72), (1, 480, 640)])
def test_fp16_backbone_error_is_that_of_its_semantics(shape):
    model, _, _ = util.build_model(dict(CASES[0]), DEV)
    img = B.image(shape, 21)
    with torch.no_grad():
        ex = copy.deepcopy(model.backbone).double()(img.double())
        emu = B.forward_f64(model.backbone, img)
    got = B.backbone_forward(_tc(model), img)[1:]
    stats = {}
    for g, e, x, name in zip(got, emu, ex, ("coarse", "fine")):
        g = g.permute(0, 3, 1, 2).double()
        scale = x.abs().max().item()
        err, err_emu = (g - x).abs().max().item(), (e - x).abs().max().item()
        stats.update({f"{name}_scale": scale, f"{name}_err_kernel": err, f"{name}_err_emulation": err_emu,
                      f"{name}_kernel_vs_emulation": (g - e).abs().max().item()})
        assert err <= 2 * err_emu + 1e-6 * scale, f"{name}: {err:.3e} vs emulation {err_emu:.3e} (scale {scale:.3e})"
    util.record("backbone_fp16_%dx%dx%d" % shape, stats)


def _convs(w):
    return [*w.l1, *w.l2, w.l2_down, *w.l3, w.l3_down, w.l3_out, w.l2_out, *w.l2_out2, w.l1_out, *w.l1_out2]


def test_fp16_pack_equals_split_weight_hi():
    """The fp16 pack (torch's round to nearest even of w * 2^e) holds exactly the hi planes of the split pack
    (split_weight, the library's split kernel), main and remainder, and no lo plane."""
    from loftr_b200.loftr import TensorCoreBackbone
    model, _, _ = util.build_model(dict(CASES[0]), DEV)
    w16, k16 = _tc(model)._pack()
    ws, ks = TensorCoreBackbone(model.backbone)._pack()
    p16 = {t.data_ptr(): t for t in k16 if t is not None}
    ps = {t.data_ptr(): t for t in ks if t is not None}
    for a, b in zip(_convs(w16), _convs(ws)):
        assert a.w_lo is None and a.wr_lo is None and b.w_lo is not None
        assert torch.equal(p16[a.w_hi], ps[b.w_hi])
        assert (a.wr_hi is None) == (b.wr_hi is None)
        if b.wr_hi is not None:
            assert torch.equal(p16[a.wr_hi], ps[b.wr_hi])
        assert torch.equal(p16[a.scale], ps[b.scale]) and torch.equal(p16[a.shift], ps[b.shift])


def test_fp16_backbone_ignores_channel_padding_and_repeats_bitwise():
    """196-channel planes have a row stride of 200; channels 196..199 are never written.  A NaN-filled workspace gives
    the bits of a zeroed one, and a repeated run gives the same bits."""
    model, _, _ = util.build_model(dict(CASES[0]), DEV)
    tc = _tc(model)
    img = B.image((2, 96, 136), 12)
    _, zc, zf = B.backbone_forward(tc, img, 0)
    _, nc, nf = B.backbone_forward(tc, img, 0xFF)
    assert torch.isfinite(nc).all() and torch.isfinite(nf).all()
    assert torch.equal(zc, nc) and torch.equal(zf, nf)
    _, rc, rf = B.backbone_forward(tc, img, 0)
    assert torch.equal(zc, rc) and torch.equal(zf, rf)


def test_fp16_backbone_image_alone_equals_image_in_batch():
    model, _, _ = util.build_model(dict(CASES[0]), DEV)
    tc = _tc(model)
    batch = B.image((16, 136, 200), 13)
    _, bc, bf = B.backbone_forward(tc, batch)
    for i in (0, 7, 15):
        _, c, f = B.backbone_forward(tc, batch[i:i + 1].contiguous())
        assert torch.equal(c[0], bc[i]) and torch.equal(f[0], bf[i]), i


# ---------------------------------------------------------------------------------------------- end to end
def _model(case, backbone_impl="b200_fp16"):
    return util.build_model(case, DEV, backbone_impl)[0]


@pytest.mark.parametrize("name", ["ds_thr0", "ds_masked_scaled", "ds_unequal", "ds_empty", "ot_thr0"])
def test_fp16_matcher_runs_every_path(name):
    """matcher(batch), forward_static and CapturedMatcher with the fp16 backbone: the split mode's keys, dtypes and
    (b, i) order; the static and captured outputs equal the eager forward bit for bit."""
    case = _CASE[name]
    inp = util.device_inputs(case)
    model = _model(case)
    got = util.eager(model, inp)
    ref = util.eager(_model(case, "b200"), inp)
    assert list(got) == list(ref)
    for k, v in ref.items():
        if torch.is_tensor(v):
            assert got[k].dtype == v.dtype and got[k].shape[1:] == v.shape[1:], k
    pairs = list(zip(got["b_ids"].tolist(), got["i_ids"].tolist()))
    assert pairs == sorted(pairs)
    m = got["b_ids"].shape[0]
    if name == "ds_empty":
        assert m == 0
    st = dict(inp)
    model.forward_static(st)
    assert int(st["num_matches"].item()) == m
    for k in LIST_KEYS:
        assert torch.equal(st[k][:m], got[k]), f"forward_static {k}"
    masked = "mask0" in inp
    cm = loftr_b200.CapturedMatcher(model, case["n"], case["hw0"], case["hw1"], masks=masked, scales="scale0" in inp)
    cap = dict(inp)
    cm(cap)
    for k, v in got.items():
        if torch.is_tensor(v):
            assert torch.equal(cap[k], v), f"CapturedMatcher {k}"
    util.record("backbone_fp16_matcher_" + name, {"matches": m, "matches_split": int(ref["b_ids"].shape[0])})


def test_fp16_bank_equals_stacked_forward_and_is_refused_by_the_split_mode():
    model = _model(_CASE["ds_thr0"])
    split = _model(_CASE["ds_thr0"], "b200")
    inp = build_inputs({"n": 3, "hw0": (240, 320), "hw1": (240, 320), "images": "smooth", "iseed": 1})
    imgs = torch.from_numpy(np.concatenate([inp["image0"], inp["image1"]])).to(DEV)
    idx0 = torch.tensor([0, 1, 2, 2, 3, 5], device=DEV)
    idx1 = torch.tensor([1, 0, 3, 3, 3, 2], device=DEV)
    bank = model.extract_features(imgs)
    got = model.match_features(bank, idx0, bank, idx1)
    ref = {"image0": imgs[idx0], "image1": imgs[idx1]}
    model(ref)
    ref = {k: v for k, v in ref.items() if k not in ("image0", "image1")}
    assert list(got) == list(ref)
    for k, v in ref.items():
        if torch.is_tensor(v):
            assert torch.equal(got[k], v), k
        else:
            assert got[k] == v, k
    assert got["b_ids"].shape[0] > 0
    with pytest.raises(RuntimeError, match="other backbone weights"):
        split.match_features(bank, idx0, bank, idx1)
    with pytest.raises(RuntimeError, match="other backbone weights"):
        model.match_features(split.extract_features(imgs), idx0, bank, idx1)


def test_fp16_agreement_with_split_backbone_at_8x640x480():
    """Recorded, not gated: with random weights the coarse logits reach 70-105 (SURVEY.md hard part 1), which
    exaggerates the effect of fp16 features on the match list.  No trained checkpoint is available here."""
    case = BASELINE_CASES["b8"]
    inp = util.device_inputs(case)
    got = util.eager(_model(case), inp)
    ref = util.eager(_model(case, "b200"), inp)
    kg = {k: n for n, k in enumerate(zip(*(got[x].tolist() for x in ("b_ids", "i_ids", "j_ids"))))}
    kr = {k: n for n, k in enumerate(zip(*(ref[x].tolist() for x in ("b_ids", "i_ids", "j_ids"))))}
    common = sorted(set(kg) & set(kr))
    ig = torch.tensor([kg[k] for k in common], dtype=torch.long, device=DEV)
    ir = torch.tensor([kr[k] for k in common], dtype=torch.long, device=DEV)
    stats = {"matches_fp16": len(kg), "matches_split": len(kr), "shared": len(common),
             "overlap": len(common) / max(len(kg), len(kr), 1)}
    if common:
        rel = ((got["mconf"][ig] - ref["mconf"][ir]).abs() / ref["mconf"][ir].abs().clamp_min(1e-30)).double()
        dxy = (got["mkpts1_f"][ig] - ref["mkpts1_f"][ir]).abs().amax(1).double()
        stats.update({"mconf_rel_max": rel.max().item(), "mconf_rel_median": rel.median().item(),
                      "mkpts1_f_max_px": dxy.max().item(), "mkpts1_f_median_px": dxy.median().item()})
    util.record("backbone_fp16_vs_split_b8_640x480", stats)
    assert stats["matches_fp16"] > 0
