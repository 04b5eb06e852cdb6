"""The single-pass fp16 matching mode (`match_precision="fp16"`: lb_coarse_match_fp16, lb_transformer_forward_fp16) at
the tile, chunk, split and mask boundaries of tests/test_kernel_edges_gpu.py, through the same harness.

Coarse matching: the match list follows ref64.coarse_match of the fp16 emulation's conf_matrix (match-list rule of
DESIGN.md §5, the emulation's top-2 as adjudicator), and conf_matrix follows the emulation elementwise at rtol 1e-3.

Transformers: one `self` and one `cross` layer, so a rounding flip of one layer cannot spread through later ones.
Each output is held to max|kernel - emu64| <= 4 max|emu32 - emu64| + 1e-6 scale, where emu64 / emu32 are the fp16
emulation run in float64 / float32 (test_kernel_edges_gpu._bound16; tests/test_match_fp16_rule_cpu.py shows which
defects this rule sees), and to the 2x contract of DESIGN.md §16 against exact float64."""
import numpy as np
import pytest
import torch

import loftr_b200.loftr as LM
import ref64 as R
import test_kernel_edges_gpu as E
from test_kernel_edges_gpu import (BLOCK_M, CM_SHAPES, COARSE_TF, DS_PARAMS, FULL_ONLY, OT_PARAMS, WINDOWS, _cdiv,
                                   _feats, _sms, _t, cm_launch, kv_splits)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP16 = "fp16"
LAYERS = ("self", "cross")


def _model(coarse="linear", fine="linear"):
    return E._model(coarse=coarse, fine=fine, precision=FP16, layer_names=LAYERS)[0]


# ------------------------------------------------------------------------------------------------ coarse matching
@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
@pytest.mark.parametrize("case", CM_SHAPES)
def test_fp16_coarse_matching_shapes(case, match_type):
    _, _, _, _, stats = E._run_cm(case, match_type, f"fp16_cm_{match_type}", precision=FP16)
    assert stats["n"] > 0 or case["hw0c"] == (1, 1) or match_type == "sinkhorn"


@pytest.mark.parametrize("case", OT_PARAMS)
def test_fp16_sinkhorn_parameters(case):
    E._run_cm(case, "sinkhorn", "fp16_cm_sinkhorn_params", precision=FP16)


@pytest.mark.parametrize("case", DS_PARAMS)
def test_fp16_dual_softmax_parameters(case):
    _, _, _, _, stats = E._run_cm(case, "dual_softmax", "fp16_cm_dual_softmax_params", precision=FP16)
    assert stats["n"] > 0


@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
def test_fp16_conf_matrix_multi_chunk(match_type):
    case = {"n": 2, "hw0c": (12, 20), "hw1c": (40, 60), "border_rm": 2}
    assert cm_launch(2, 240, 2400, _sms())["n_chunks"] > 1
    E._run_cm(case, match_type, f"fp16_cm_conf_matrix_{match_type}", precision=FP16)


# ------------------------------------------------------------------------------------------------ transformers
def coarse_gemm_items(n, L, S, attention):
    """Work items (128-row x 256-column tiles) of every tensor-core GEMM of one coarse layer's passes, from a mirror of
    engine.cu's gemm_shape: linear attention runs the k|v projection per source group and the attention epilogue per
    query group, full attention its q and k|v projections over all rows; merge, MLP1 and MLP2 run over all rows."""
    tiles = lambda batches, rows, cols: batches * _cdiv(rows, BLOCK_M) * _cdiv(cols, 256)
    items = []
    for xr, sr in ((L, S), (S, L)):   # cross passes; a self pass over both sets has more rows
        if attention == "linear":
            items += [tiles(n, sr, 512), tiles(n, xr, 256)]
        else:
            items += [tiles(1, n * xr, 256), tiles(1, n * sr, 512)]
        items += [tiles(1, n * xr, 256), tiles(1, n * xr, 512), tiles(1, n * xr, 256)]
    return items


COARSE_TF16 = COARSE_TF + [pytest.param({"n": 11, "L": 4800, "S": 4800, "ctas_tiles": 3}, id="n11_L4800_S4800")]


@pytest.mark.parametrize("attention", ["linear", "full"])
@pytest.mark.parametrize("case", COARSE_TF16)
def test_fp16_coarse_transformer_shapes(case, attention):
    n, L, S = case["n"], case["L"], case["S"]
    if "ctas_tiles" in case:   # every persistent CTA of every coarse GEMM runs at least 3 tiles
        sms = _sms()
        assert min(coarse_gemm_items(n, L, S, attention)) >= case["ctas_tiles"] * sms
    f0, f1 = _feats(n, L, S, 256, 31)
    E._tf_check(f"fp16_tf_coarse_{attention}_n{n}_L{L}_S{S}", _model(coarse=attention).loftr_coarse, attention, f0,
                f1, precision=FP16)


@pytest.mark.parametrize("case", FULL_ONLY)
def test_fp16_full_attention_key_tiles(case):
    n, L, S = case["n"], case["L"], case["S"]
    f0, f1 = _feats(n, L, S, 256, 37)
    m0 = m1 = None
    if "key_hole" in case:
        m0, m1 = np.ones((n, L), bool), np.ones((n, S), bool)
        m1[:, case["key_hole"][0]:case["key_hole"][1]] = False
    E._tf_check(f"fp16_tf_coarse_full_{n}_{L}_{S}_{case.get('key_hole')}", _model(coarse="full").loftr_coarse, "full",
                f0, f1, m0, m1, precision=FP16)


@pytest.mark.parametrize("attention", ["linear", "full"])
def test_fp16_coarse_transformer_split_k(attention):
    sms = _sms()
    assert kv_splits(2, 200, sms) > 1 and kv_splits(67, 200, sms) == 1
    tf = _model(coarse=attention).loftr_coarse
    f0, f1 = _feats(2, 200, 200, 256, 41)
    E._tf_check(f"fp16_tf_coarse_{attention}_n2_200", tf, attention, f0, f1, precision=FP16)
    reps = _cdiv(67, 2)
    f0b, f1b = np.tile(f0, (reps, 1, 1))[:67], np.tile(f1, (reps, 1, 1))[:67]
    E._tf_check(f"fp16_tf_coarse_{attention}_n67_200_splits1", tf, attention, f0b, f1b, precision=FP16)


@pytest.mark.parametrize("attention", ["linear", "full"])
def test_fp16_coarse_transformer_fully_masked_images(attention):
    n, L, S = 3, 130, 97
    f0, f1 = _feats(n, L, S, 256, 43)
    rs = np.random.RandomState(44)
    m0, m1 = rs.uniform(size=(n, L)) > 0.2, rs.uniform(size=(n, S)) > 0.3
    m1[1] = False
    m0[2] = False
    E._tf_check(f"fp16_tf_coarse_{attention}_fully_masked", _model(coarse=attention).loftr_coarse, attention, f0, f1,
                m0, m1, precision=FP16)


@pytest.mark.parametrize("attention", ["linear", "full"])
@pytest.mark.parametrize("case", WINDOWS)
def test_fp16_window_transformer(case, attention):
    tf = _model(fine=attention).loftr_fine
    f0, f1 = _feats(case["n"], case["l"], case["s"], 128, 47)
    if attention == "full" and case["l"] != case["s"]:
        with pytest.raises(RuntimeError, match="equal window sizes"):   # built for equal windows only
            tf(_t(f0), _t(f1))
        return
    E._tf_check(f"fp16_tf_fine_{attention}_n{case['n']}_{case['l']}x{case['s']}", tf, attention, f0, f1,
                precision=FP16)


@pytest.mark.parametrize("attention", ["linear", "full"])
@pytest.mark.parametrize("live", [4001, 0])
def test_fp16_window_transformer_live_bound(live, attention):
    """5003 windows of capacity, `live` of them computed: 4001 x 9 rows end inside a 128-row tile of each set, 0
    computes nothing.  The live rows follow the emulation.  Every row of the token state (fp32 features and both planes,
    scratch columns included) keeps its bits past the end of the last 128-row tile that holds live rows; the rows
    between the live count and that tile's end are computed on capacity memory that nothing reads (DESIGN.md §11)."""
    n, ww, c = 5003, 9, 128
    rows = live * ww
    tile_end = _cdiv(rows, BLOCK_M) * BLOCK_M
    assert live == 0 or rows < tile_end < n * ww
    tf = _model(fine=attention).loftr_fine
    f0, f1 = (_t(f) for f in _feats(n, ww, ww, c, 53))
    st = LM._TokenState(n * ww, n * ww, c, DEV)
    st.x[: n * ww] = f0.reshape(-1, c)
    st.x[n * ww:] = f1.reshape(-1, c)
    st.cat_hi.zero_()
    st.cat_lo.zero_()
    LM.split_planes(st.x, st.cat_hi, st.cat_lo, 0)
    before = [t.clone() for t in (st.x, st.cat_hi, st.cat_lo)]
    tf.run(st, n, ww, ww, None, torch.tensor([live], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    for what, t, b in zip(("x", "cat_hi", "cat_lo"), (st.x, st.cat_hi, st.cat_lo), before):
        for base in (0, n * ww):
            assert torch.equal(t[base + tile_end:base + n * ww], b[base + tile_end:base + n * ww]), \
                f"{what}: a row past the last live tile of the set at row {base} changed"
    if live == 0:
        return
    g0, g1 = (x[:live] for x in st.sides(n, ww, ww))
    lw = R.layer_weights(tf, DEV)
    lw32 = R.layer_weights(tf, DEV, dtype=torch.float32)
    x0, x1 = f0[:live], f1[:live]
    exact = R.transformer(x0.double(), x1.double(), lw, LAYERS, 8, attention=attention)
    e64 = R.transformer(x0.double(), x1.double(), lw, LAYERS, 8, attention=attention, fp16=True)
    e32 = R.transformer(x0, x1, lw32, LAYERS, 8, attention=attention, fp16=True)
    name = f"fp16_tf_fine_{attention}_live{live}_of_{n}"
    finding = E.RATIO_FINDINGS.get(name)
    E._bound16(name + "_feat0", g0, e64[0], e32[0], exact[0], finding)
    E._bound16(name + "_feat1", g1, e64[1], e32[1], exact[1], finding)
