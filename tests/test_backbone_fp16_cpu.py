"""CPU-side checks of the fp16 backbone (`backbone_impl="b200_fp16"`): the float64 emulation's structure, the weight
pack (hi planes only), the workspace size, the constructor refusals and the library version gate."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import loftr_b200
import backbone_ref as B
import util
from cases import CASES
from loftr_b200 import _lib
from loftr_b200.loftr import TensorCoreBackbone, weight_exponent


def _model():
    model, _, _ = util.build_model(dict(CASES[0]), "cpu")
    return model


def test_emulation_without_rounding_is_the_float64_module():
    m = _model().backbone
    rs = np.random.RandomState(3)
    img = torch.from_numpy(rs.uniform(0, 1, (2, 1, 32, 48)).astype(np.float32))
    with torch.no_grad():
        ex_c, ex_f = copy.deepcopy(m).double()(img.double())
        got_c, got_f = B.forward_f64(m, img, fp16=False)
    for got, ex in ((got_c, ex_c), (got_f, ex_f)):
        assert got.shape == ex.shape
        assert (got - ex).abs().max().item() <= 1e-12 * ex.abs().max().item()


def test_emulation_rounds_like_fp16():
    """With rounding the emulation differs from the float64 module at the level of fp16, not more."""
    m = _model().backbone
    rs = np.random.RandomState(4)
    img = torch.from_numpy(rs.uniform(0, 1, (1, 1, 32, 32)).astype(np.float32))
    with torch.no_grad():
        ex_c, ex_f = copy.deepcopy(m).double()(img.double())
        got_c, got_f = B.forward_f64(m, img)
    for got, ex in ((got_c, ex_c), (got_f, ex_f)):
        rel = (got - ex).abs().max().item() / ex.abs().max().item()
        assert 1e-5 < rel < 3e-2, rel


def _conv_weights(w):
    """(name, LbConvWeights, conv module) of every convolution after the stem."""
    out = [(f"l{i}[{j}]", getattr(w, f"l{i}")[j]) for i in (1, 2, 3) for j in range(4)]
    out += [("l2_down", w.l2_down), ("l3_down", w.l3_down), ("l3_out", w.l3_out), ("l2_out", w.l2_out),
            ("l2_out2[0]", w.l2_out2[0]), ("l2_out2[1]", w.l2_out2[1]), ("l1_out", w.l1_out),
            ("l1_out2[0]", w.l1_out2[0]), ("l1_out2[1]", w.l1_out2[1])]
    return out


def _modules(m):
    mods = {f"l{i}[{2 * b + c}]": getattr(getattr(m, f"layer{i}")[b], f"conv{c + 1}")
            for i in (1, 2, 3) for b in range(2) for c in range(2)}
    mods.update({"l2_down": m.layer2[0].downsample[0], "l3_down": m.layer3[0].downsample[0],
                 "l3_out": m.layer3_outconv, "l2_out": m.layer2_outconv, "l2_out2[0]": m.layer2_outconv2[0],
                 "l2_out2[1]": m.layer2_outconv2[3], "l1_out": m.layer1_outconv, "l1_out2[0]": m.layer1_outconv2[0],
                 "l1_out2[1]": m.layer1_outconv2[3]})
    return mods


def test_fp16_pack_holds_the_hi_planes_only():
    """Every packed plane is fp16(w * 2^e) in the tap-major layout (main channels, then the 16-channel remainder
    planes of the 196-channel inputs), with split_weight's exponent e; no lo plane is packed."""
    m = _model().backbone
    w, keep = TensorCoreBackbone(m, precision="fp16")._build()
    by_ptr = {t.data_ptr(): t for t in keep if t is not None}
    mods = _modules(m)
    lib = _lib.load()
    rem_layers = 0
    for name, cw in _conv_weights(w):
        assert cw.w_lo is None and cw.wr_lo is None, name
        wt = mods[name].weight.detach().float()
        cout, cin, k, _ = wt.shape
        e = weight_exponent(wt)
        tap = wt.permute(0, 2, 3, 1).reshape(cout, k * k, cin)
        cbl, rc = C.c_int(), C.c_int()
        _lib.check(lib.lb_conv_layout(cin, C.byref(cbl), C.byref(rc)))
        cmain = cbl.value * 64
        main = torch.zeros(cout, k * k, cmain)
        main[:, :, :min(cin, cmain)] = tap[:, :, :cmain]
        hi = by_ptr[cw.w_hi]
        assert hi.dtype == torch.float16 and torch.equal(hi, (main.reshape(cout, -1) * 2.0 ** e).half()), name
        assert cw.scale and by_ptr[cw.scale].dtype == torch.float32
        if cmain < cin:
            rem_layers += 1
            rem = torch.zeros(cout, k * k, 16)
            rem[:, :, :cin - cmain] = tap[:, :, cmain:]
            assert torch.equal(by_ptr[cw.wr_hi], (rem.reshape(cout, -1) * 2.0 ** e).half()), name
        else:
            assert cw.wr_hi is None, name
    assert rem_layers == 8   # every convolution that reads a 196-channel activation
    assert lib.lb_version() >= _lib.BACKBONE_FP16_VERSION


def test_fp16_workspace_is_about_half():
    m = _model().backbone
    w, _ = TensorCoreBackbone(m, precision="fp16")._build()
    lib = _lib.load()
    for n, h, wd in ((1, 480, 640), (16, 480, 640), (8, 136, 200)):
        split = lib.lb_backbone_workspace_bytes(C.byref(w), n, h, wd)
        fp16 = lib.lb_backbone_workspace_bytes_fp16(C.byref(w), n, h, wd)
        assert 0.49 < fp16 / split < 0.51, (n, h, wd, split, fp16)
    util.record("backbone_fp16_workspace_16x480x640", {
        "split_bytes": lib.lb_backbone_workspace_bytes(C.byref(w), 16, 480, 640),
        "fp16_bytes": lib.lb_backbone_workspace_bytes_fp16(C.byref(w), 16, 480, 640)})


def test_constructor_modes_and_refusals():
    cfg = loftr_b200.get_cfg("indoor_ds")
    assert loftr_b200.LoFTR(cfg).backbone_impl == "b200"            # "auto" is unchanged
    model = loftr_b200.LoFTR(cfg, backbone_impl="b200_fp16")
    assert model.backbone_impl == "b200_fp16" and model._tc_backbone.precision == "fp16"
    assert model._bank_key()[0] == "b200_fp16"    # a bank records the mode it was extracted in
    with pytest.raises(ValueError):
        TensorCoreBackbone(model.backbone, precision="bf16")
    with pytest.raises(ValueError):
        loftr_b200.LoFTR(cfg, backbone_impl="fp16")
    cfg64 = copy.deepcopy(cfg)
    cfg64["resnetfpn"]["initial_dim"] = 64                            # a 64-channel stem: not built
    with pytest.raises(ValueError, match="tensor-core backbone"):
        loftr_b200.LoFTR(cfg64, backbone_impl="b200_fp16")


def test_fp16_backbone_refuses_an_older_library(monkeypatch):
    util.old_library(monkeypatch, 107)
    assert _lib.BACKBONE_FP16_VERSION == 108
    with pytest.raises(RuntimeError, match=r"version 108 or newer.*is version 107"):
        loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds"), backbone_impl="b200_fp16")
    loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds"), backbone_impl="b200")   # the other modes need nothing new


def test_fp16_entry_points_are_bound():
    lib = _lib.load()
    for name in ("lb_backbone_workspace_bytes_fp16", "lb_backbone_forward_fp16"):
        assert _lib.SIGNATURES[name][1] == getattr(lib, name).argtypes
