"""Full (softmax) attention without a GPU: the oracle against the reference's goldens, the masked-row convention, the
model's configuration surface and the library-version guard of the binding."""
import numpy as np
import pytest

import loftr_b200
import util
from full_cases import FA_MODULE_CASE, FULL_CASES, build_fa_module_inputs
from loftr_b200 import _lib
from loftr_b200.loftr import LocalFeatureTransformer, LoFTREncoderLayer
from oracle import loftr_oracle as O


@pytest.mark.parametrize("case", FULL_CASES, ids=[c["name"] for c in FULL_CASES])
def test_full_oracle_matches_reference(case):
    gold = util.load_golden(case["name"])
    out = util.oracle_forward(case)
    np.testing.assert_allclose(out["feat_c0"][:, ::7, ::5], gold["feat_c0_s"], rtol=2e-4, atol=2e-4)
    np.testing.assert_allclose(out["feat_c1"][:, ::7, ::5], gold["feat_c1_s"], rtol=2e-4, atol=2e-4)
    stats = util.compare_matches(out, gold, gold, conf_rtol=1e-3, px_tol=0.05, label=case["name"])
    assert stats["n"] == len(gold["b_ids"]) or stats["overlap"] >= 0.995
    m = len(gold["b_ids"])
    if m and len(out["b_ids"]) == m and (out["i_ids"] == gold["i_ids"]).all():
        nf = gold["fine_tf0"].shape[0]
        np.testing.assert_allclose(out["expec_f"], gold["expec_f"], atol=2e-3)
        np.testing.assert_allclose(out["feat_f0_unfold"][:nf], gold["fine_tf0"], rtol=1e-3, atol=1e-3)
        np.testing.assert_allclose(out["feat_f1_unfold"][:nf], gold["fine_tf1"], rtol=1e-3, atol=1e-3)


def test_full_attention_masked_module_convention():
    """Valid rows equal the reference's FullAttention; the reference's padded rows are NaN, ours are 0."""
    gold = util.load_golden(FA_MODULE_CASE["name"])
    q, k, v, qm, km = build_fa_module_inputs()
    out = O.full_attention(q, k, v, qm, km)
    assert np.isfinite(out).all()
    assert np.isnan(gold["out"][~qm]).all()          # what the convention replaces
    np.testing.assert_allclose(out[qm], gold["out"][qm], rtol=1e-5, atol=1e-6)
    assert (out[~qm] == 0).all()
    # a row whose keys are all masked gets a zero message too; unmasked calls are a plain softmax
    km0 = km.copy()
    km0[0] = False
    assert (O.full_attention(q, k, v, qm, km0)[0] == 0).all()
    plain = O.full_attention(q[:1, :5], k[:1], v[:1])
    s = np.einsum("lhd,shd->lhs", q[0, :5].astype(np.float64), k[0].astype(np.float64)) / np.sqrt(q.shape[-1])
    a = np.exp(s - s.max(-1, keepdims=True))
    a /= a.sum(-1, keepdims=True)
    np.testing.assert_allclose(plain[0], np.einsum("lhs,shd->lhd", a, v[0].astype(np.float64)), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("coarse", ["linear", "full"])
@pytest.mark.parametrize("fine", ["linear", "full"])
def test_loftr_builds_every_attention_combination(coarse, fine):
    cfg = loftr_b200.get_cfg("indoor_ds")
    cfg["coarse"]["attention"], cfg["fine"]["attention"] = coarse, fine
    m = loftr_b200.LoFTR(cfg)
    assert {l.attention for l in m.loftr_coarse.layers} == {coarse}
    assert {l.attention for l in m.loftr_fine.layers} == {fine}
    ref = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).state_dict()
    sd = m.state_dict()
    assert list(sd) == list(ref)
    assert all(sd[k].shape == ref[k].shape for k in sd)
    m.load_state_dict(ref)   # a linear model's checkpoint loads into a full model and back


@pytest.mark.parametrize("bad", ["softmax", "Full", None])
def test_unknown_attention_is_rejected(bad):
    with pytest.raises(ValueError):
        LoFTREncoderLayer(256, 8, bad)
    cfg = loftr_b200.get_cfg("indoor_ds")
    cfg["fine"]["attention"] = bad
    with pytest.raises(ValueError):
        loftr_b200.LoFTR(cfg)


def test_binding_refuses_full_attention_on_an_old_library(monkeypatch):
    util.old_library(monkeypatch, 101)
    assert _lib.MIN_VERSION == 101 and _lib.FULL_ATTENTION_VERSION == 102
    cfg = dict(loftr_b200.get_cfg("indoor_ds")["coarse"], attention="full")
    tf = LocalFeatureTransformer(cfg)
    with pytest.raises(RuntimeError, match=r"102.*version 101"):
        tf.run(object(), 1, 4, 4)
    # linear layers do not need the newer library: the guard is not what stops them
    lin = LocalFeatureTransformer(dict(cfg, attention="linear"))
    with pytest.raises(AttributeError):
        lin.run(object(), 1, 4, 4)


def test_layer_kinds_match_the_header():
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "loftr_b200.h")).read()
    kinds = dict(re.findall(r"#define LB_(LAYER_\w+) (\d+)", hdr))
    assert {k: int(v) for k, v in kinds.items()} == {"LAYER_SELF": _lib.LAYER_SELF, "LAYER_CROSS": _lib.LAYER_CROSS,
                                                     "LAYER_SELF_FULL": _lib.LAYER_SELF_FULL,
                                                     "LAYER_CROSS_FULL": _lib.LAYER_CROSS_FULL}
