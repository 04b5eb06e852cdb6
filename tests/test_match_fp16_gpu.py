"""The single-pass fp16 matching mode (`match_precision="fp16"`: lb_transformer_forward_fp16, lb_coarse_match_fp16) on
the GPU.

Per output, the error against float64 (ref64) is held to twice the error of the float64 emulation of the same
semantics (ref64 with fp16=True) plus 1e-6 of the output's scale, as for the fp16 backbone.  The coarse match list
follows the emulation's by the match-list rule of DESIGN.md §5 with the emulation in place of fp64.  Every public path
runs unchanged on top, bit for bit against the eager forward, and the bits do not depend on the workspace's contents
or on repetition."""
import ctypes as C

import numpy as np
import pytest
import torch

import loftr_b200
import loftr_b200.loftr as L
import ref64
import util
from cases import BASELINE_CASES, CASES, build_cfg, build_inputs
from loftr_b200 import _lib
from match_cap_ref import LIST_KEYS, apply_cap, capped_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_CASE = {c["name"]: c for c in CASES}


def _bound(name, got, emu, exact, stats):
    scale = exact.abs().max().item()
    err, err_emu = (got.double() - exact).abs().max().item(), (emu - exact).abs().max().item()
    stats.update({f"{name}_scale": scale, f"{name}_err_kernel": err, f"{name}_err_emulation": err_emu,
                  f"{name}_kernel_vs_emulation": (got.double() - emu).abs().max().item()})
    assert err <= 2 * err_emu + 1e-6 * scale, f"{name}: {err:.3e} vs emulation {err_emu:.3e} (scale {scale:.3e})"


def _tf(d_model, attention, seed):
    torch.manual_seed(seed)
    cfg = {"d_model": d_model, "nhead": 8, "layer_names": ["self", "cross"] * 2, "attention": attention}
    tf = L.LocalFeatureTransformer(cfg, precision="fp16").eval()
    return cfg, tf.to(DEV), ref64.layer_weights(tf, DEV)


def _run(tf, f0, f1, mask=None, live=None, fill=None):
    """LocalFeatureTransformer.run on a fresh token state; fill: byte pattern of the workspace (None: torch.empty)."""
    n, l, c = f0.shape
    s = f1.shape[1]
    st = L._TokenState(n * l, n * s, c, DEV)
    st.x[: n * l] = f0.reshape(-1, c)
    st.x[n * l:] = f1.reshape(-1, c)
    L.split_planes(st.x, st.cat_hi, st.cat_lo, 0)
    if fill is None:
        tf.run(st, n, l, s, mask, live)
    else:
        lib = _lib.load()
        arr, kinds, _ = tf._pack()
        nbytes = lib.lb_transformer_workspace_bytes(c, 8, n, l, s)
        ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=DEV)
        sts = _lib.LbTransformerState(st.x.data_ptr(), st.cat_hi.data_ptr(), st.cat_lo.data_ptr(), _lib.ptr(mask), n,
                                      l, s, _lib.ptr(live))
        _lib.check(lib.lb_transformer_forward_fp16(arr, kinds, len(tf.layers), c, 8, C.byref(sts), ws.data_ptr(),
                                                   nbytes, L._stream(st.x)))
    torch.cuda.synchronize()
    a, b = st.sides(n, l, s)
    return a.clone(), b.clone()


# ---------------------------------------------------------------------------------------------- transformers
@pytest.mark.parametrize("attention", ["linear", "full"])
@pytest.mark.parametrize("masked", [False, True])
def test_coarse_transformer_error_is_that_of_its_semantics(attention, masked):
    cfg, tf, layers = _tf(256, attention, seed=11)
    n, l, s = 2, 300, 170          # L != S, partial tiles
    g = torch.Generator().manual_seed(3)
    f0 = (torch.randn(n, l, 256, generator=g) + 0.5).to(DEV)
    f1 = (torch.randn(n, s, 256, generator=g) + 0.5).to(DEV)
    m0 = m1 = mask = None
    if masked:
        m0 = torch.ones(n, l, dtype=torch.bool, device=DEV)
        m1 = torch.ones(n, s, dtype=torch.bool, device=DEV)
        m0[0, 250:] = False
        m1[1, 100:] = False
        mask = torch.cat([m0.reshape(-1), m1.reshape(-1)]).to(torch.uint8)
    got = _run(tf, f0, f1, mask)
    x0, x1 = f0.double(), f1.double()
    exact = ref64.transformer(x0, x1, layers, cfg["layer_names"], 8, m0, m1, attention)
    emu = ref64.transformer(x0, x1, layers, cfg["layer_names"], 8, m0, m1, attention, fp16=True)
    stats = {}
    for name, gg, e, x in zip(("feat0", "feat1"), got, emu, exact):
        _bound(name, gg, e, x, stats)
    util.record(f"match_fp16_coarse_tf_{attention}{'_masked' if masked else ''}", stats)


@pytest.mark.parametrize("ww", [25, 9])
@pytest.mark.parametrize("attention", ["linear", "full"])
@pytest.mark.parametrize("live", [None, 37])
def test_fine_transformer_error_is_that_of_its_semantics(ww, attention, live):
    cfg, tf, layers = _tf(128, attention, seed=12)
    n = 150                        # windows per set (the capacity when `live` bounds them)
    g = torch.Generator().manual_seed(4)
    f0 = (torch.randn(n, ww, 128, generator=g) * 2).to(DEV)
    f1 = (torch.randn(n, ww, 128, generator=g) * 2).to(DEV)
    lv = None if live is None else torch.tensor([live], dtype=torch.int32, device=DEV)
    got = _run(tf, f0, f1, live=lv)
    k = n if live is None else live
    x0, x1 = f0[:k].double(), f1[:k].double()
    exact = ref64.transformer(x0, x1, layers, cfg["layer_names"], 8, attention=attention)
    emu = ref64.transformer(x0, x1, layers, cfg["layer_names"], 8, attention=attention, fp16=True)
    stats = {}
    for name, gg, e, x in zip(("feat0", "feat1"), got, emu, exact):
        _bound(name, gg[:k], e, x, stats)
    util.record(f"match_fp16_fine_tf_{attention}_{ww}{'' if live is None else '_live'}", stats)


def test_transformer_bits_do_not_depend_on_the_workspace_or_repetition():
    for d_model, attention, shape in ((256, "linear", (2, 300, 170)), (256, "full", (2, 300, 170)),
                                      (128, "linear", (64, 25, 25))):
        _, tf, _ = _tf(d_model, attention, seed=13)
        n, l, s = shape
        f0 = torch.randn(n, l, d_model, device=DEV)
        f1 = torch.randn(n, s, d_model, device=DEV)
        a = _run(tf, f0, f1, fill=0)
        for fill in (0xFF, 0):     # 0xFF: every fp16 / fp32 of the workspace is NaN
            b = _run(tf, f0, f1, fill=fill)
            assert all(torch.equal(x, y) for x, y in zip(a, b)), (d_model, attention, fill)


# ---------------------------------------------------------------------------------------------- coarse matching
def _cm_inputs(n, h, w, seed, masked):
    rs = np.random.RandomState(seed)
    base = rs.standard_normal((n, h * w, 256)).astype(np.float32)
    f0 = base * 1.2 + 3.0          # a large common-mode part like the real features (SURVEY.md §7 hard part 1)
    perm = rs.permutation(h * w)
    f1 = (base[:, perm] * 1.2 + 3.0 + 0.3 * rs.standard_normal((n, h * w, 256))).astype(np.float32)
    f0, f1 = torch.from_numpy(f0).to(DEV), torch.from_numpy(f1).to(DEV)
    m0 = m1 = None
    if masked:
        m0 = torch.ones(n, h, w, dtype=torch.bool, device=DEV)
        m1 = torch.ones(n, h, w, dtype=torch.bool, device=DEV)
        m0[0, :, w - 7:] = False
        m1[-1, h - 5:] = False
    return f0, f1, m0, m1


def _coarse(match_type, f0, f1, m0, m1, h, w, k=None):
    cfg = build_cfg({"thr": 0.0})["match_coarse"]
    cfg.update(match_type=match_type, return_conf_matrix=True, skh_prefilter=False, max_matches_per_pair=k)
    mod = L.CoarseMatching(cfg, precision="fp16").eval().to(DEV)
    data = {"hw0_i": (h * 8, w * 8), "hw1_i": (h * 8, w * 8), "hw0_c": (h, w), "hw1_c": (h, w)}
    mod(f0, f1, data, None if m0 is None else m0.flatten(-2), None if m1 is None else m1.flatten(-2))
    torch.cuda.synchronize()
    return mod, data


@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
@pytest.mark.parametrize("masked", [False, True])
def test_conf_matrix_and_match_list_follow_the_emulation(match_type, masked):
    n, h, w = 2, 30, 40
    f0, f1, m0, m1 = _cm_inputs(n, h, w, 5, masked)
    mod, data = _coarse(match_type, f0, f1, m0, m1, h, w)
    mc = mod.config
    bs = mod.bin_score.detach().double() if match_type == "sinkhorn" else None
    fm0 = None if m0 is None else m0.flatten(-2)
    fm1 = None if m1 is None else m1.flatten(-2)
    exact = ref64.conf_matrix(f0.double(), f1.double(), mc, fm0, fm1, bs)
    emu = ref64.conf_matrix(f0.double(), f1.double(), mc, fm0, fm1, bs, fp16=True)
    got = data["conf_matrix"]
    if masked:   # cells whose row and column are both padding: 0 in the engine (DESIGN.md §5)
        valid = (fm0[:, :, None] | fm1[:, None, :]).double()
        got, exact, emu = got * valid, exact * valid, emu * valid
    stats = {}
    _bound("conf_matrix", got, emu, exact, stats)
    ref = ref64.coarse_match(emu, mc, data["hw0_i"], (h, w), (h, w), m0, m1)
    r2, c2 = ref64.top2(emu)
    gold = {"row_top2_f64": r2.cpu().numpy(), "col_top2_f64": c2.cpu().numpy()}
    g = {k: data[k].cpu().numpy() for k in ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c")}
    r = {k: v.cpu().numpy() for k, v in ref.items()}
    stats.update(util.compare_matches(g, r, gold, conf_rtol=1e-3, px_tol=1e-3, min_overlap=0.995,
                                      label=f"{match_type} masked={masked}"))
    util.record(f"match_fp16_coarse_{match_type}{'_masked' if masked else ''}", stats)
    assert stats["n"] > 0


def test_coarse_match_bits_do_not_depend_on_the_workspace_and_the_cap_keeps_rows(monkeypatch):
    n, h, w = 3, 30, 40
    f0, f1, m0, m1 = _cm_inputs(n, h, w, 6, True)
    keys = ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c")
    _, a = _coarse("dual_softmax", f0, f1, m0, m1, h, w)
    _, b = _coarse("dual_softmax", f0, f1, m0, m1, h, w)
    for key in keys + ("conf_matrix",):
        assert torch.equal(a[key], b[key]), key
    for k in (1, 17):
        _, capped = _coarse("dual_softmax", f0, f1, m0, m1, h, w, k=k)
        rows = capped_rows(a["b_ids"], a["mconf"], k)
        for key in keys:
            assert torch.equal(capped[key], a[key][rows]), (k, key)
    real_empty = torch.empty

    def nan_workspace(*size, **kw):   # the only uint8 buffer of CoarseMatching.run is its workspace: 0xFF = NaN
        t = real_empty(*size, **kw)
        return t.fill_(255) if kw.get("dtype") is torch.uint8 else t

    monkeypatch.setattr(torch, "empty", nan_workspace)
    _, c = _coarse("dual_softmax", f0, f1, m0, m1, h, w)
    for key in keys + ("conf_matrix",):
        assert torch.equal(a[key], c[key]), key


# ---------------------------------------------------------------------------------------------- end to end
def _model(case, backbone_impl="b200", match_precision="fp16"):
    return util.build_model(case, DEV, backbone_impl, match_precision)[0]


@pytest.mark.parametrize("name", ["ds_thr0", "ds_masked_scaled", "ds_unequal", "ds_empty", "ot_thr0"])
def test_fp16_matching_runs_every_path(name):
    """matcher(batch), forward_static, CapturedMatcher and a capped run in fp16 matching mode: the split mode's keys,
    dtypes and (b, i) order; static, captured and repeated outputs equal the eager forward bit for bit; a capped run
    equals the selected rows of the uncapped one."""
    case = _CASE[name]
    inp = util.device_inputs(case)
    model = _model(case)
    got = util.eager(model, inp)
    ref = util.eager(_model(case, match_precision="split"), inp)
    assert list(got) == list(ref)
    for k, v in ref.items():
        if torch.is_tensor(v):
            assert got[k].dtype == v.dtype and got[k].shape[1:] == v.shape[1:], k
    pairs = list(zip(got["b_ids"].tolist(), got["i_ids"].tolist()))
    assert pairs == sorted(pairs)
    m = got["b_ids"].shape[0]
    if name == "ds_empty":
        assert m == 0
    again = util.eager(model, inp)
    for k, v in got.items():
        if torch.is_tensor(v):
            assert torch.equal(again[k], v), f"repeat {k}"
    st = dict(inp)
    model.forward_static(st)
    assert int(st["num_matches"].item()) == m
    for k in LIST_KEYS:
        assert torch.equal(st[k][:m], got[k]), f"forward_static {k}"
    cm = loftr_b200.CapturedMatcher(model, case["n"], case["hw0"], case["hw1"], masks="mask0" in inp,
                                    scales="scale0" in inp)
    cap = dict(inp)
    cm(cap)
    for k, v in got.items():
        if torch.is_tensor(v):
            assert torch.equal(cap[k], v), f"CapturedMatcher {k}"
    if m:
        k = max(1, m // (2 * case["n"]))
        model.coarse_matching.max_matches_per_pair = k
        capped = util.eager(model, inp)
        sel = apply_cap(got, k)
        for key in LIST_KEYS:
            assert torch.equal(capped[key], sel[key]), f"cap {k}: {key}"
    util.record("match_fp16_matcher_" + name, {"matches": m, "matches_split": int(ref["b_ids"].shape[0])})


def test_fp16_matching_bank_equals_stacked_forward():
    model = _model(_CASE["ds_thr0"])
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


@pytest.mark.parametrize("backbone", ["b200", "b200_fp16"])
def test_fp16_matching_agreement_with_split_at_8x640x480(backbone):
    """Recorded, not gated: with random weights the coarse logits reach 70-105 (SURVEY.md hard part 1), which
    exaggerates the effect of fp16 products on the match list.  No trained checkpoint is available here."""
    case = BASELINE_CASES["b8"]
    inp = util.device_inputs(case)
    got = util.eager(_model(case, backbone), inp)
    ref = util.eager(_model(case, backbone, "split"), inp)
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
    util.record(f"match_fp16_vs_split_{backbone}_b8_640x480", stats)
    assert stats["matches_fp16"] > 0
