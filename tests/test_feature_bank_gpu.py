"""Pair lists matched from per-image feature banks (`LoFTR.extract_features` / `LoFTR.match_features`).

`match_features` must write what `matcher(batch)` writes for the explicitly stacked batch of the same pairs.  The
tensor-core backbone computes every output pixel with the same instructions whatever else is in the batch, and every
stage after it sees the same pair-major inputs, so with `backbone_impl="b200"` every key is compared bit for bit.
cuDNN may pick other algorithms for another batch shape, so the PyTorch backbone is held to the match-list rule of
DESIGN.md §5 instead."""
import numpy as np
import pytest
import torch

import loftr_b200
import util
import weights as W
from cases import BASELINE_CASES, build_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_INPUT_KEYS = ("image0", "image1", "mask0", "mask1", "scale0", "scale1")
# pair list over a bank of 6 images: a repeated pair (2, 3), a self pair (3, 3), both orders of (0, 1)
IDX0 = [0, 1, 2, 2, 3, 4, 5]
IDX1 = [1, 0, 3, 3, 3, 5, 2]


def _model(name="indoor_ds", thr=0.0, backbone_impl="auto", attention="linear", conf_matrix=False, wseed=0):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = loftr_b200.get_cfg(name, thr=thr)
    cfg["coarse"]["attention"] = cfg["fine"]["attention"] = attention
    if conf_matrix:
        cfg["match_coarse"]["return_conf_matrix"] = True
    model = loftr_b200.LoFTR(cfg, backbone_impl=backbone_impl).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict({k: torch.from_numpy(v) for k, v in W.make_state(shapes, seed=wseed).items()})
    return model.to(DEV)


def _images(k, hw, seed=1, images="smooth"):
    """k seeded images [k, 1, H, W] on the device (the image0 and image1 halves of a build_inputs case)."""
    inp = build_inputs({"n": (k + 1) // 2, "hw0": hw, "hw1": hw, "images": images, "iseed": seed})
    return torch.from_numpy(np.concatenate([inp["image0"], inp["image1"]])[:k]).to(DEV)


def _idx(v, dtype=torch.int64):
    return torch.tensor(v, dtype=dtype, device=DEV)


def _forward(model, imgs0, idx0, imgs1, idx1, masks=None, scales=None):
    """matcher(batch) on the stacked pairs -> the keys it wrote, in order."""
    i0, i1 = idx0.long(), idx1.long()
    batch = {"image0": imgs0[i0], "image1": imgs1[i1]}
    if masks is not None:
        batch["mask0"], batch["mask1"] = masks[0][i0], masks[1][i1]
    if scales is not None:
        batch["scale0"], batch["scale1"] = scales[0][i0], scales[1][i1]
    model(batch)
    return {k: v for k, v in batch.items() if k not in _INPUT_KEYS}


def _assert_bitwise(got, ref, label):
    assert list(got) == list(ref), f"{label}: keys {list(got)} vs {list(ref)}"
    for k, v in ref.items():
        if torch.is_tensor(v):
            assert got[k].dtype == v.dtype and got[k].shape == v.shape, (label, k, got[k].shape, v.shape)
            assert torch.equal(got[k], v), f"{label}: {k} differs from matcher(batch)"
        else:
            assert got[k] == v, (label, k, got[k], v)
    assert got["mkpts0_f"] is got["mkpts0_c"]


def _assert_match_list_rule(got, ref, label):
    assert list(got) == list(ref), label
    for k, v in ref.items():
        if not torch.is_tensor(v):
            assert got[k] == v, (label, k)
        else:
            assert got[k].dtype == v.dtype, (label, k)
    np_ = lambda d: {k: d[k].cpu().numpy() for k in ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c",
                                                     "mkpts0_f", "mkpts1_f")}
    return util.compare_matches(np_(got), np_(ref), None, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995, label=label)


def _run_pair_lists(model, hw=(480, 640), hw_other=(384, 512), exact=True, label=""):
    """One bank of 6 images, matched over IDX0 x IDX1, plus pairs across two banks of different image sizes."""
    imgs = _images(6, hw)
    other = _images(3, hw_other, seed=5, images="rand")
    bank = model.extract_features(imgs)
    bank_other = model.extract_features(other)
    check = _assert_bitwise if exact else _assert_match_list_rule
    counts = []
    for lab, b0, im0, i0, b1, im1, i1 in (
            ("one bank", bank, imgs, _idx(IDX0), bank, imgs, _idx(IDX1, torch.int32)),
            ("two sizes", bank, imgs, _idx([0, 3, 3, 5]), bank_other, other, _idx([1, 0, 2, 2])),
            ("two sizes swapped", bank_other, other, _idx([2, 0]), bank, imgs, _idx([4, 4]))):
        got = model.match_features(b0, i0, b1, i1)
        ref = _forward(model, im0, i0, im1, i1)
        check(got, ref, f"{label} {lab}")
        counts.append(int(got["b_ids"].shape[0]))
    util.record("feature_bank_" + label, {"matches": counts})
    return counts


@pytest.mark.parametrize("name,thr", [("indoor_ds", 0.0), ("indoor_ds", 0.2), ("indoor_ot", 0.0)],
                         ids=["indoor_ds-thr0", "indoor_ds-thr0.2", "indoor_ot-thr0"])
def test_pair_list_equals_stacked_forward_bitwise(name, thr):
    counts = _run_pair_lists(_model(name, thr), label=f"{name}_thr{thr}")
    if thr == 0.0:
        assert min(counts) > 0
    else:   # no confidence of these seeded weights reaches 0.2: the M = 0 path
        assert max(counts) == 0


def test_full_attention_pair_list_equals_stacked_forward_bitwise():
    counts = _run_pair_lists(_model(attention="full"), hw=(240, 320), hw_other=(256, 192), label="full_attention")
    assert min(counts) > 0


def test_conf_matrix_pair_list_equals_stacked_forward_bitwise():
    model = _model(conf_matrix=True)
    _run_pair_lists(model, hw=(240, 320), hw_other=(192, 256), label="conf_matrix")


def test_outdoor_832_masks_and_scales_bitwise():
    """outdoor_ds at 832x832, a different padding mask per image and per-image scales, gathered per pair."""
    case = BASELINE_CASES["out4"]
    inp = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in build_inputs(case).items()}
    imgs = torch.cat([inp["image0"], inp["image1"]])
    masks = torch.cat([inp["mask0"], inp["mask1"]])
    scales = torch.cat([inp["scale0"], inp["scale1"]])
    model = _model("outdoor_ds", 0.0)
    bank = model.extract_features(imgs, masks)
    idx0, idx1 = _idx([0, 1, 2, 7, 3, 3]), _idx([4, 5, 6, 0, 3, 7])
    got = model.match_features(bank, idx0, bank, idx1, scales, scales)
    ref = _forward(model, imgs, idx0, imgs, idx1, (masks, masks), (scales, scales))
    _assert_bitwise(got, ref, "outdoor 832 masked scaled")
    assert got["b_ids"].shape[0] > 0
    util.record("feature_bank_outdoor832", {"matches": int(got["b_ids"].shape[0])})


def test_torch_backbone_pair_list_follows_the_match_list_rule():
    _run_pair_lists(_model(backbone_impl="torch"), hw=(240, 320), hw_other=(192, 256), exact=False,
                    label="torch_backbone")


def test_bank_layout():
    for impl in ("b200", "torch"):
        model = _model(backbone_impl=impl)
        imgs = _images(3, (96, 128))
        bank = model.extract_features(imgs)
        assert len(bank) == 3 and tuple(bank.hw_i) == (96, 128) and tuple(bank.hw_c) == (12, 16)
        assert tuple(bank.hw_f) == (48, 64) and bank.mask is None
        assert bank.feat_c.shape == (3, 256, 12, 16) and bank.feat_f.shape == (3, 128, 48, 64)
        channels_last = bank.feat_f.stride(1) == 1
        assert channels_last == (impl == "b200"), impl


def test_errors_and_empty_list():
    model = _model()
    imgs = _images(4, (96, 128))
    bank = model.extract_features(imgs)
    ok = _idx([0, 1])
    with pytest.raises(IndexError, match=r"`idx1` holds indices in \[0, 4\], outside the bank's \[0, 4\)"):
        model.match_features(bank, ok, bank, _idx([0, 4]))
    with pytest.raises(IndexError, match="outside"):
        model.match_features(bank, _idx([-1, 0]), bank, ok)
    with pytest.raises(TypeError, match="int32 or int64"):
        model.match_features(bank, ok.float(), bank, ok)
    with pytest.raises(TypeError, match="int32 or int64"):
        model.match_features(bank, [0, 1], bank, ok)
    with pytest.raises(ValueError, match="is on cpu"):
        model.match_features(bank, ok.cpu(), bank, ok)
    with pytest.raises(ValueError, match="same length"):
        model.match_features(bank, ok, bank, _idx([0]))
    with pytest.raises(ValueError, match="scale0 and scale1 together"):
        model.match_features(bank, ok, bank, ok, scale0=torch.ones(4, 2, device=DEV))
    with pytest.raises(ValueError, match=r"must be \[4, 2\]"):
        model.match_features(bank, ok, bank, ok, torch.ones(2, 2, device=DEV), torch.ones(4, 2, device=DEV))
    masked = model.extract_features(imgs, torch.ones(4, 12, 16, dtype=torch.bool, device=DEV))
    with pytest.raises(ValueError, match="both banks carry masks or neither"):
        model.match_features(masked, ok, bank, ok)
    with pytest.raises(ValueError, match="no images"):
        model.extract_features(imgs[:0])
    with pytest.raises(ValueError, match="masks must be"):
        model.extract_features(imgs, torch.ones(4, 12, 15, dtype=torch.bool, device=DEV))
    with pytest.raises(TypeError, match="ImageFeatures"):
        model.match_features(imgs, ok, bank, ok)

    # an empty pair list: the outputs of a forward without matches
    full = model.match_features(bank, ok, bank, ok)
    empty = model.match_features(bank, _idx([]), bank, _idx([]))
    assert list(empty) == list(full) and empty["bs"] == 0
    for k, v in full.items():
        if torch.is_tensor(v):
            assert empty[k].shape == (0,) + tuple(v.shape[1:]) and empty[k].dtype == v.dtype, k

    # results land in a caller-provided dict
    mine = {"frame": 7}
    assert model.match_features(bank, ok, bank, ok, data=mine) is mine and mine["frame"] == 7 and "b_ids" in mine


def test_bank_is_tied_to_the_backbone_weights():
    model = _model()
    imgs = _images(2, (96, 128))
    bank = model.extract_features(imgs)
    idx = _idx([0, 1])
    before = model.match_features(bank, idx, bank, idx.flip(0))
    model.load_state_dict(_model(wseed=0).state_dict())   # the same values, loaded again
    with pytest.raises(RuntimeError, match="other backbone weights"):
        model.match_features(bank, idx, bank, idx.flip(0))
    after = model.match_features(model.extract_features(imgs), idx, model.extract_features(imgs), idx.flip(0))
    _assert_bitwise(after, before, "re-extracted")
    with torch.no_grad():
        model.backbone.conv1.weight.mul_(1.0)   # an in-place update bumps the version
    with pytest.raises(RuntimeError, match="other backbone weights"):
        model.match_features(bank, idx, bank, idx)
