"""CPU checks of the single-pass fp16 matching mode (`match_precision="fp16"`, DESIGN.md §16): the float64 emulation
(`fp16=True` of tests/ref64.py) on hand cases, and the Python API (constructor
values, read-only attributes, the library version gate, the C entry points' argument check)."""
import copy
import ctypes as C

import pytest
import torch

import loftr_b200
import ref64 as R
import util
from loftr_b200 import _lib
from loftr_b200.loftr import CoarseMatching, LocalFeatureTransformer

F64 = torch.float64
TINY = 2.0 ** -12    # below half an fp16 ulp of values in [1, 2): rounds away


def _layers(d_model, attention, n_layers=2, seed=0):
    torch.manual_seed(seed)
    cfg = {"d_model": d_model, "nhead": 8, "layer_names": ["self", "cross"][:n_layers], "attention": attention}
    return cfg, R.layer_weights(LocalFeatureTransformer(cfg))


# ------------------------------------------------------------------------------------------------ hand cases
def test_roundings_of_one_value():
    x = torch.tensor([1.0 + TINY, 1.0 + 2.0 ** -10, 1.0 / 3.0], dtype=F64)
    assert R.r16(x).tolist() == [1.0, 1.0 + 2.0 ** -10, float(torch.tensor(1.0 / 3.0).half())]
    assert torch.equal(R.r16(x, False), x)
    w = torch.tensor([1e-3 / 3.0], dtype=F64)    # e = 21: fp16(w * 2^21) keeps 11 bits of w whatever its magnitude
    assert R.w16(w, 21).item() == float(torch.tensor(1e-3 / 3.0 * 2.0 ** 21).half()) * 2.0 ** -21
    assert abs(R.w16(w, 21).item() / w.item() - 1) < 2.0 ** -11 and R.w16(w, 21).item() != w.item()


def test_linear_attention_rounds_k_and_v():
    # K = elu(k)+1 = 1 + TINY and V = 1 + TINY round to 1: the rounded message equals the one of K = V = 1
    q = torch.randn(1, 5, 2, 4, dtype=F64)
    k = torch.full((1, 7, 2, 4), TINY, dtype=F64)
    v = torch.full((1, 7, 2, 4), 1.0 + TINY, dtype=F64)
    exact1 = R.linear_attention(q, torch.zeros_like(k), torch.ones_like(v))
    assert torch.allclose(R.linear_attention(q, k, v, fp16=True), exact1, rtol=1e-15, atol=0)
    assert not torch.allclose(R.linear_attention(q, k, v), exact1, rtol=1e-6, atol=0)


def test_full_attention_rounds_q_k_v_and_p():
    q = torch.full((1, 3, 1, 32), 1.0 + TINY, dtype=F64)
    k = torch.full((1, 4, 1, 32), 1.0 + TINY, dtype=F64)
    v = torch.arange(4, dtype=F64).view(1, 4, 1, 1).expand(1, 4, 1, 32) * (1.0 + TINY)
    one = R.full_attention(torch.ones_like(q), torch.ones_like(k), v.half().double())
    assert torch.allclose(R.full_attention(q, k, v, fp16=True), one, rtol=1e-15, atol=0)   # equal logits: mean fp16(V)
    # P = exp(S / sqrt(D) - rowmax) is rounded in P V, not in the row sum
    a = 2.0 ** -4
    qq = torch.zeros(1, 1, 1, 32, dtype=F64)
    qq[..., 0] = 1.0
    kk = torch.zeros(1, 2, 1, 32, dtype=F64)
    kk[0, 1, 0, 0] = a
    vv = torch.cat([torch.ones(1, 1, 1, 32), torch.full((1, 1, 1, 32), 2.0)], 1).double()
    p0 = torch.exp(torch.tensor(-a / 32 ** 0.5, dtype=F64))
    assert R.r16(p0) != p0
    want = (R.r16(p0) * 1.0 + 2.0) / (p0 + 1.0)
    assert torch.allclose(R.full_attention(qq, kk, vv, fp16=True), torch.full((1, 1, 1, 32), want.item(), dtype=F64),
                          rtol=1e-15, atol=0)
    assert not torch.allclose(R.full_attention(qq, kk, vv), torch.full((1, 1, 1, 32), want.item(),
                                                                                       dtype=F64), rtol=1e-9, atol=0)


def test_encoder_layer_rounds_activations_and_weights_but_not_the_residual():
    cfg, layers = _layers(256, "linear", n_layers=1, seed=3)
    w = layers[0]
    x0 = (torch.randn(1, 9, 256, dtype=F64) + 3.0).half().double()        # fp16 values in about [1, 6]
    x = x0 * (1.0 + TINY / 8)                                            # rounds back to x0 everywhere it is an operand
    out0, out = R.encoder_layer(x0, x0, w, 8, fp16=True), R.encoder_layer(x, x, w, 8, fp16=True)
    assert torch.allclose(out - x, out0 - x0, rtol=0, atol=1e-12)        # only the exact residual sees the change
    exact = R.encoder_layer(x, x, w, 8) - R.encoder_layer(x0, x0, w, 8)
    assert (exact - (x - x0)).abs().max() > 1e-7
    # weights within a fraction of an fp16 ulp of their hi plane give the same layer
    e = R.layer_exponents(w)
    keys = {"q_proj.weight": "qkv", "k_proj.weight": "qkv", "v_proj.weight": "qkv", "merge.weight": "merge",
            "mlp.0.weight": "mlp0", "mlp.2.weight": "mlp2"}
    w_hi = dict(w, **{k: R.w16(w[k], e[g]) for k, g in keys.items()})
    w_near = dict(w_hi, **{k: w_hi[k] * (1.0 + TINY / 4) for k in keys})
    assert R.layer_exponents(w_near) == e
    assert torch.equal(R.encoder_layer(x0, x0, w_near, 8, fp16=True), R.encoder_layer(x0, x0, w_hi, 8, fp16=True))
    assert not torch.equal(R.encoder_layer(x0, x0, w_near, 8), R.encoder_layer(x0, x0, w_hi, 8))


def test_score_matrix_rounds_both_features():
    mc = loftr_b200.get_cfg("indoor_ds")["match_coarse"]
    f0 = (torch.randn(1, 6, 256, dtype=F64) + 2).half().double()
    f1 = (torch.randn(1, 5, 256, dtype=F64) + 2).half().double()
    near = R.conf_matrix(f0 * (1 + TINY / 8), f1 * (1 - TINY / 8), mc, fp16=True)
    assert torch.equal(near, R.conf_matrix(f0, f1, mc, fp16=True))
    assert not torch.equal(R.conf_matrix(f0 * (1 + TINY / 8), f1, mc), R.conf_matrix(f0, f1, mc, fp16=True))


# ------------------------------------------------------------------------------------------------ Python API
def test_constructor_modes():
    cfg = loftr_b200.get_cfg("indoor_ds")
    assert loftr_b200.LoFTR(cfg).match_precision == "split"       # the default is unchanged
    for backbone in ("b200", "b200_fp16"):
        for prec in ("split", "fp16"):
            m = loftr_b200.LoFTR(cfg, backbone_impl=backbone, match_precision=prec)
            assert m.backbone_impl == backbone and m.match_precision == prec
            assert m.loftr_coarse.precision == m.loftr_fine.precision == m.coarse_matching.precision == prec
    m = loftr_b200.LoFTR(cfg, match_precision="fp16")
    assert m.backbone_impl == "b200"                               # "auto" does not follow match_precision
    assert set(m.state_dict()) == set(loftr_b200.LoFTR(cfg).state_dict())
    for obj, attr in ((m, "match_precision"), (m.loftr_coarse, "precision"), (m.coarse_matching, "precision")):
        with pytest.raises(AttributeError):
            setattr(obj, attr, "split")
    assert LocalFeatureTransformer(cfg["coarse"], precision="fp16").precision == "fp16"
    assert CoarseMatching(cfg["match_coarse"], precision="fp16").precision == "fp16"


@pytest.mark.parametrize("bad", ["FP16", "bf16", "fp32", "", None, 16, ["fp16"]])
def test_bad_precisions_are_rejected(bad):
    cfg = loftr_b200.get_cfg("indoor_ds")
    with pytest.raises(ValueError, match="match_precision"):
        loftr_b200.LoFTR(cfg, match_precision=bad)
    with pytest.raises(ValueError, match="precision"):
        LocalFeatureTransformer(cfg["coarse"], precision=bad)
    with pytest.raises(ValueError, match="precision"):
        CoarseMatching(cfg["match_coarse"], precision=bad)


def test_fp16_matching_refuses_an_older_library(monkeypatch):
    util.old_library(monkeypatch, 108)
    assert _lib.MATCH_FP16_VERSION == 109
    cfg = loftr_b200.get_cfg("indoor_ds")
    with pytest.raises(RuntimeError, match=r"match_precision.*version 109 or newer.*is version 108"):
        loftr_b200.LoFTR(cfg, match_precision="fp16")
    for make in (lambda: LocalFeatureTransformer(cfg["fine"], precision="fp16"),
                 lambda: CoarseMatching(cfg["match_coarse"], precision="fp16")):
        with pytest.raises(RuntimeError, match=r"version 109 or newer.*is version 108"):
            make()
    loftr_b200.LoFTR(copy.deepcopy(cfg), backbone_impl="b200_fp16")   # the split matching needs nothing new


def test_fp16_entry_points_and_the_gemm_hook_are_bound_and_check_arguments():
    lib = _lib.load()
    assert lib.lb_version() == _lib.GEMM_FP16_VERSION > _lib.MATCH_FP16_VERSION
    for name in ("lb_transformer_forward_fp16", "lb_coarse_match_fp16", "lb_gemm_fp16"):
        assert _lib.SIGNATURES[name][1] == getattr(lib, name).argtypes
    assert lib.lb_gemm_fp16(None, None, 64, 0, None, None, 64, 0, None, 80, 0, 1, 128, 80, 64, None) != 0
    assert b"lb_gemm_fp16: N must be a multiple of 32" in lib.lb_last_error()
    a = _lib.LbCoarseMatchArgs()
    for k in (-1, -7):
        assert lib.lb_coarse_match_fp16(C.byref(a), k, None, 0, None) != 0
        assert b"max_per_pair must be 0" in lib.lb_last_error()
