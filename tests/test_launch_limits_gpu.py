"""The matcher at its launch-size limits: 65,535 pairs in one call, and buffers past 2^31 elements.

Launch dimensions of engine.cu that grow with the caller's data (CUDA: grid.x <= 2^31 - 1, grid.y / grid.z <= 65,535):

| launch                                   | grid                                  | grows with          | limit and where it is held                       |
|------------------------------------------|---------------------------------------|---------------------|--------------------------------------------------|
| full_attn_wgmma_kernel (coarse, full)    | (cdiv(L, 128), 8, images of the pass) | pairs               | z: lb_transformer_forward refuses n > 65,535;     |
| kv_gemm_kernel (coarse, linear)          | (splits, 2, images of the pass)       | pairs               | a self pass over both sets (2n images) runs only |
|                                          |                                       |                     | for 2n <= 65,535, else one pass per set          |
| coarse_prep_kernel                       | (cdiv(h*w, 32), cdiv(C, 32), n_out)   | pairs               | z: lb_coarse_prep(_indexed) refuses n_out > 65,535 |
| preprocess_images_kernel                 | (cdiv(W, 128), cdiv(H, 8), n)         | images              | z: lb_preprocess_images (existing check)         |
| rectify_images_kernel                    | (cdiv(W, 128), cdiv(H, 8), n)         | pairs * candidates  | z: lb_rectify_images, check_rectify_candidates   |
| geometry_score_kernel                    | (hypothesis tiles, B)                 | pairs               | y: lb_estimate_geometry (existing check)         |
| unpack_matches_kernel                    | (cdiv(capacity, 256), world)          | ranks               | y: world size, not a reachable case              |
| gemm_split_kernel, conv3x3_halo_kernel,  | min(work items, SMs)                  | -                   | persistent: bounded by the SM count              |
| conv_stem7x7_tc_kernel                   |                                       |                     |                                                  |
| window_attn_kernel, window_full_attn_... | min(windows, 3 or 4 * SMs)            | -                   | grid-stride: bounded by the SM count             |
| split_planes_kernel                      | min(total / 256 + 1, 4096)            | -                   | grid-stride                                      |
| kv_tile_merge_kernel                     | cdiv(n * 8 * 1056, 256)               | pairs               | x: n <= 65,535 keeps it below 2.2e6 blocks       |
| mask_extent, bin_lse, match_cap kernels  | n                                     | pairs               | x                                                |
| rectify_search_kernel                    | n / K                                 | pairs               | x                                                |
| mask_term, fill, lse_merge, argmax_merge,| cdiv(n * L or n * S, 256)             | cells               | x: 2^31 blocks are 5.5e11 cells; the coarse      |
| ot_dead, match_flag, match_count/scatter |                                       |                     | workspace alone would take > 100 TB              |
| coarse_query_kernel<side>                | cdiv(n * Q, 256)                      | queries             | x: likewise unreachable                          |
| fine_gather(_vec8)_kernel                | 2M                                    | windows             | x: M >= 2^30 needs > 250 TB of fine state        |
| fine_bias_kernel, fine_match_kernel      | cdiv(2M, 8), cdiv(M, 8)               | windows             | x: likewise                                      |
| rectify_points, epipolar_error, pack     | cdiv(m, 256)                          | points / matches    | x: likewise                                      |
| geometry_compact / refit kernels         | B                                     | pairs               | x                                                |

Before this file the coarse transformer's self pass put 2n images in grid.z, so any call of more than 32,767 pairs of
equal-size images failed after the backbone with cudaErrorInvalidConfiguration.  The pair limit is now 65,535 per
call (loftr.MAX_PAIRS), refused by the Python API before the backbone (test_launch_limits_cpu.py) and by the C
entries before any launch.

65,535 pairs: the outputs equal, bit for bit, the same pairs run in chunks of 4,096.  Each pair's backbone, transformer
rows, coarse rows and windows depend on that pair alone (DESIGN.md §12), and with S <= 256 the score passes take one
column chunk (pick_chunks) whatever the pair count, and kv_splits gives one split above 66 images: no summation order
depends on the pair count at these shapes.

Past 2^31 elements: conf_matrix (n = 6, L = S = 19,200: n*L*S = 2.21e9) against float64 elementwise, and the fine
stage at M = 167,800 windows, where the fine-state planes [2*M*WW, 2*Cf] hold 2.148e9 elements, against float64 by the
dense-output rule of test_kernel_edges_gpu.py.  Every test states its expected peak memory (from the buffer shapes),
records the measured one through util.record and is skipped when the device has less free memory than that plus
2 GiB."""
import numpy as np
import pytest
import torch

import ref64 as R
import util
from cases import CASES, build_cfg, build_cm_inputs
from oracle import loftr_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GiB = 2 ** 30
LIMIT = 65535
CHUNK = 4096
LIST = ("b_ids", "i_ids", "j_ids", "m_bids", "gt_mask", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f",
        "expec_f")
QUERY = ("q_i_ids", "q_j_ids", "qconf", "qmutual", "qvalid", "qinside", "qpts0_f", "qpts1_c", "qpts1_f", "qexpec_f")


def _budget(name, peak):
    """Skips unless the device has `peak` bytes free plus 2 GiB; then starts the peak count."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < peak + 2 * GiB:
        pytest.skip(f"{name}: needs {peak / GiB:.1f} GiB free plus 2 GiB of margin, the device has {free / GiB:.1f}")
    torch.cuda.reset_peak_memory_stats()


def _record(name, peak, **stats):
    util.record(name, {"peak_expected_gib": peak / GiB, "peak_measured_gib": torch.cuda.max_memory_allocated() / GiB,
                       **stats})


def _model(attention="linear", cap=1):
    """thr 0 and no border: every pair keeps its mutual matches; at most `cap` per pair bounds the fine stage."""
    model, _, _ = util.build_model({"thr": 0.0, "border_rm": 0, "coarse_attention": attention}, DEV)
    model.coarse_matching.max_matches_per_pair = cap
    return model


def _images(n, hw, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.rand(n, 1, *hw, generator=g, device=DEV)


def _chunked(call, n, keys, pair_keys=()):
    """call(s, e) -> output dict of pairs [s, e), over chunks of CHUNK pairs -> the concatenated outputs, with the
    pair ids of `pair_keys` offset to the whole list."""
    parts = []
    for s in range(0, n, CHUNK):
        out = call(s, min(s + CHUNK, n))
        parts.append({k: out[k] + s if k in pair_keys else out[k] for k in keys})
    return {k: torch.cat([p[k] for p in parts]) for k in keys}


def _refused(call, who):
    """call() with 65,536 pairs raises ValueError before anything is launched."""
    from loftr_b200 import _lib
    lib = _lib.load()
    launches = lib.lb_launch_count()
    with pytest.raises(ValueError, match=rf"{who}: 65536 pairs exceed the 65535 pairs of one call"):
        call()
    assert lib.lb_launch_count() == launches


# ------------------------------------------------------------------------------------------------ 65,535 pairs
@pytest.mark.parametrize("attention", ["linear", "full"])
def test_forward_65535_pairs_equals_chunks(attention):
    """8x8 images (one coarse cell, 4x4 fine maps), 65,535 pairs; one match per pair.
    Expected peak: the coarse transformer's workspace holds K^T V partials for 8 splits of every image of a pass,
    2 * 65,535 * 8 heads * 8 * 1,056 floats = 33.0 GiB (with either attention; one split is used at this count),
    plus the coarse token state and the pair outputs: 40 GiB.  The fine state of 65,535 windows (about 218 KB each,
    13.6 GiB) comes after that workspace is freed."""
    peak = 40 * GiB
    _budget("forward_65535", peak)
    model = _model(attention)
    im0, im1 = _images(LIMIT, (8, 8), 1), _images(LIMIT, (8, 8), 2)
    whole = util.eager(model, {"image0": im0, "image1": im1})
    assert whole["b_ids"].shape[0] == LIMIT   # one cell each, conf 1 > thr
    ref = _chunked(lambda s, e: util.eager(model, {"image0": im0[s:e], "image1": im1[s:e]}), LIMIT, LIST,
                   ("b_ids", "m_bids"))
    util.assert_same(whole, ref, LIST, f"forward 65535 {attention}")
    _record(f"forward_65535_{attention}", peak, matches=int(whole["b_ids"].shape[0]))
    del whole, ref
    one = torch.cat([im0, im0[:1]])
    _refused(lambda: model({"image0": one, "image1": one}), "forward")
    _refused(lambda: model.forward_static({"image0": one, "image1": one}), "forward_static")


@pytest.mark.parametrize("attention", ["linear", "full"])
def test_match_features_65535_pairs_equals_chunks(attention):
    """A bank of four 16x16 images (2x2 coarse cells), 65,535 index pairs over its 16 ordered pairs; one match per
    pair at most.  Expected peak: as the forward test, 40 GiB (the coarse state of 2 * 65,535 * 4 tokens adds 1 GiB).
    """
    peak = 40 * GiB
    _budget("match_features_65535", peak)
    model = _model(attention)
    bank = model.extract_features(_images(4, (16, 16), 3))
    k = torch.arange(LIMIT, device=DEV)
    idx0, idx1 = k % 4, (k // 4) % 4
    whole = model.match_features(bank, idx0, bank, idx1)
    assert whole["b_ids"].shape[0] > LIMIT // 2, whole["b_ids"].shape
    ref = _chunked(lambda s, e: model.match_features(bank, idx0[s:e], bank, idx1[s:e]), LIMIT, LIST,
                   ("b_ids", "m_bids"))
    util.assert_same(whole, ref, LIST, f"match_features 65535 {attention}")
    _record(f"match_features_65535_{attention}", peak, matches=int(whole["b_ids"].shape[0]))
    del whole, ref
    k = torch.arange(LIMIT + 1, device=DEV) % 4
    _refused(lambda: model.match_features(bank, k, bank, k), "match_features")
    pts = torch.full((LIMIT + 1, 1, 2), 7.0, device=DEV)
    _refused(lambda: model.match_points_features(bank, k, bank, k, pts), "match_points_features")


def test_match_points_65535_pairs_equals_chunks():
    """8x8 images, 65,535 pairs of one query each (Q = 1).  Expected peak: as the forward test, 40 GiB."""
    peak = 40 * GiB
    _budget("match_points_65535", peak)
    model = _model()
    im0, im1 = _images(LIMIT, (8, 8), 4), _images(LIMIT, (8, 8), 5)
    g = torch.Generator(device=DEV).manual_seed(6)
    pts = torch.rand(LIMIT, 1, 2, generator=g, device=DEV) * 8
    whole = {"image0": im0, "image1": im1}
    model.match_points(whole, pts)
    assert bool(whole["qinside"].any())

    def chunk(s, e):
        d = {"image0": im0[s:e], "image1": im1[s:e]}
        model.match_points(d, pts[s:e])
        return d

    ref = _chunked(chunk, LIMIT, QUERY)
    util.assert_same(whole, ref, QUERY, "match_points 65535")
    _record("match_points_65535", peak)
    del whole, ref
    one = torch.cat([im0, im0[:1]])
    _refused(lambda: model.match_points({"image0": one, "image1": one}, torch.cat([pts, pts[:1]])), "match_points")


# ------------------------------------------------------------------------------------------------ past 2^31 elements
@pytest.mark.parametrize("match_type", ["dual_softmax", "sinkhorn"])
def test_conf_matrix_past_2_31_elements_vs_f64(match_type):
    """CoarseMatching with return_conf_matrix on n = 6 pairs of 120x160 cells: 6 * 19,200^2 = 2.21e9 elements.
    Pair 5's block holds element 2^31 (row 15,848) and ends the matrix.  Its rows around 2^31 and its last rows are
    compared elementwise against float64 at rtol 1e-3; the match list of all six pairs against ref64 by
    util.compare_matches.  Expected peak: conf_matrix 8.24 GiB and one pair's float64 reference, four matrices of
    2.75 GiB: 19.2 GiB, 20 GiB with the features and the workspace."""
    peak = 20 * GiB
    _budget("conf_matrix_2_31", peak)
    n, hw = 6, (120, 160)
    L = hw[0] * hw[1]
    assert n * L * L > 2 ** 31 and (n - 1) * L * L < 2 ** 31
    ot = match_type == "sinkhorn"
    inp = build_cm_inputs({"n": n, "hw0c": hw, "hw1c": hw, "amp": 3.0 if ot else 1.6, "frac": 0.6, "iseed": 23})
    mc = build_cfg({"thr": 0.0, "match_type": match_type, "border_rm": 2})["match_coarse"]
    mc["return_conf_matrix"] = True
    import loftr_b200.loftr as LM
    mod = LM.CoarseMatching(mc).eval().to(DEV)
    bin_score = 2.0
    if ot:
        mod.bin_score.data = torch.tensor(bin_score, device=DEV)
    data = {"hw0_i": (hw[0] * 8, hw[1] * 8), "hw1_i": (hw[0] * 8, hw[1] * 8), "hw0_c": hw, "hw1_c": hw}
    f0, f1 = torch.from_numpy(inp["feat_c0"]).to(DEV), torch.from_numpy(inp["feat_c1"]).to(DEV)
    mod(f0, f1, data)
    conf = data.pop("conf_matrix")
    got = {k: util.to_np(data[k]) for k in ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c")}
    refs, rows, cols = [], [], []
    straddle = 2 ** 31 // L - (n - 1) * L   # pair 5's row holding element 2^31
    stats = {}
    for b in range(n):   # float64 one pair at a time: the whole matrix would be 2.9 GB per pair
        c64 = R.conf_matrix(R.f64(f0[b:b + 1]), R.f64(f1[b:b + 1]), mc, bin_score=bin_score if ot else None)
        ref = {k: util.to_np(v) for k, v in R.coarse_match(c64, mc, data["hw0_i"], hw, hw).items()}
        ref["b_ids"] = ref["b_ids"] + b
        refs.append(ref)
        r2, c2 = R.top2(c64)
        rows.append(util.to_np(r2))
        cols.append(util.to_np(c2))
        if b == n - 1:
            for name, sl in (("straddle", slice(straddle - 8, straddle + 8)), ("last", slice(L - 16, L))):
                g, r = conf[b, sl].double(), c64[0, sl]
                big = r > 1e-30
                stats[f"{name}_rel_max"] = float(((g - r).abs() / r.clamp_min(1e-30))[big].max())
                np.testing.assert_allclose(util.to_np(g), util.to_np(r), rtol=1e-3, atol=1e-12, err_msg=name)
        del c64
    ref = {k: np.concatenate([r[k] for r in refs]) for k in refs[0]}
    gold = {"row_top2_f64": np.concatenate(rows), "col_top2_f64": np.concatenate(cols)}
    stats.update(util.compare_matches(got, ref, gold, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995,
                                      label=f"conf_matrix_2_31_{match_type}"))
    assert stats["n"] > 0
    _record(f"conf_matrix_2_31_{match_type}", peak, **stats)


M_FINE = 167_800   # 2 * M * 25 * 256 = 2.148e9 > 2^31 elements in the fine-state planes


def _windows_across(M, widths=(256, 384)):
    """The windows (side, m) whose rows hold element 2^31 of a [2*M*25, width] buffer, for each width: 256 (the fp16
    cat and MLP-hidden planes), 384 (the fp32 q|k|v rows of the window transformer)."""
    out = set()
    for w in widths:
        row = 2 ** 31 // w
        side, m = divmod(row // 25, M)
        out |= {(side, m + d) for d in (-1, 0, 1) if 0 <= m + d < M}
    return sorted(out)


def test_fine_stage_past_2_31_elements_vs_f64():
    """fine_preprocess -> loftr_fine -> FineMatching on synthetic maps at M = 167,800 windows (W = 5).  The first
    windows, those whose rows straddle element 2^31 of the planes, and the last windows are checked against float64
    by the dense-output rule.  Expected peak: token state 2*M*25 rows of 1.5 KB (12.0 GiB) + window-transformer
    workspace of 3 KB per row (24.0 GiB) = 36 GiB."""
    peak = 36 * GiB
    _budget("fine_2_31", peak)
    from test_kernel_edges_gpu import _bound
    model, _, state = util.build_model(CASES[0], DEV)
    M, W, ww = M_FINE, 5, 25
    n, hw = 1, (60, 80)
    L = hw[0] * hw[1]
    g = torch.Generator(device=DEV).manual_seed(71)
    f0, f1 = (torch.randn(n, 128, hw[0] * 4, hw[1] * 4, generator=g, device=DEV) for _ in range(2))
    c0, c1 = (torch.randn(n, L, 256, generator=g, device=DEV) for _ in range(2))
    b = torch.zeros(M, dtype=torch.int64, device=DEV)
    i, j = (torch.randint(0, L, (M,), generator=g, device=DEV) for _ in range(2))
    mk1 = torch.rand(M, 2, generator=g, device=DEV) * 600
    data = {"hw0_i": (hw[0] * 8, hw[1] * 8), "hw0_c": hw, "hw1_c": hw, "hw0_f": (hw[0] * 4, hw[1] * 4),
            "hw1_f": (hw[0] * 4, hw[1] * 4), "b_ids": b, "i_ids": i, "j_ids": j, "mkpts0_c": mk1, "mkpts1_c": mk1}
    edge = _windows_across(M)
    sel = sorted({(s, m) for s in (0, 1) for m in (0, 1, 2, M - 3, M - 2, M - 1)} | set(edge))
    ms = torch.tensor(sorted({m for _, m in sel}), device=DEV)
    fstate = model.fine_preprocess.run(f0, f1, torch.cat([c0[0], c1[0]]).contiguous(), n, L, L, data)
    p0, p1 = (x[ms].clone() for x in fstate.sides(M, ww, ww))
    model.loftr_fine.run(fstate, M, ww, ww)
    t0, t1 = fstate.sides(M, ww, ww)
    model.fine_matching(t0, t1, data)
    t0, t1 = t0[ms].clone(), t1[ms].clone()
    expec, mk1f = data["expec_f"][ms].clone(), data["mkpts1_f"][ms].clone()
    del fstate, data
    np_ = util.to_np
    bs, i_s, j_s = b[ms], i[ms], j[ms]
    fw = {k: state[f"fine_preprocess.{k}"] for k in ("down_proj.weight", "down_proj.bias", "merge_feat.weight",
                                                      "merge_feat.bias")}
    r0, r1 = R.fine_preprocess(R.f64(f0), R.f64(f1), R.f64(c0), R.f64(c1), bs, i_s, j_s, W, 4,
                               {k: R.f64(v, DEV) for k, v in fw.items()})
    o0, o1 = O.fine_preprocess(np_(f0), np_(f1), np_(c0), np_(c1), np_(bs), np_(i_s), np_(j_s), hw[1], hw[1], W, 4, fw)
    _bound("fine_2_31_preprocess_0", p0, r0, o0, extra={"windows": len(ms)})
    _bound("fine_2_31_preprocess_1", p1, r1, o1)
    tf = model.loftr_fine
    lw = R.layer_weights(tf, DEV)
    r0, r1 = R.transformer(R.f64(p0), R.f64(p1), lw, tf.layer_names, tf.nhead)
    ow = [{k: np_(v).astype(np.float32) for k, v in w.items()} for w in lw]
    o0, o1 = O.local_feature_transformer(np_(p0), np_(p1), ow, tf.layer_names, tf.nhead)
    _bound("fine_2_31_transformer_0", t0, r0, o0)
    _bound("fine_2_31_transformer_1", t1, r1, o1)
    hw_i, hw_f = (hw[0] * 8, hw[1] * 8), (hw[0] * 4, hw[1] * 4)
    re, rk = R.fine_matching(R.f64(t0), R.f64(t1), np_(mk1[ms]), bs, hw_i, hw_f)
    of = O.fine_matching(np_(t0), np_(t1), np_(mk1[ms]), np_(mk1[ms]), np_(bs), hw_i, hw_f)
    _bound("fine_2_31_expec_f", expec, re, of["expec_f"])
    _bound("fine_2_31_mkpts1_f", mk1f, rk, of["mkpts1_f"])
    _record("fine_2_31", peak, windows_checked=len(ms), straddling=str(edge))


def test_forward_static_fine_state_past_2_31_elements():
    """forward_static with capacity M_FINE on batch 2 of 96x128: its fine state is the capacity's, past 2^31 elements
    in the planes; the live prefix equals the eager forward bit for bit.  Expected peak: 36 GiB, as the fine test."""
    peak = 36 * GiB
    _budget("forward_static_2_31", peak)
    model, _, _ = util.build_model(CASES[0], DEV)
    inp = util.device_inputs(CASES[0])
    eager = util.eager(model, inp)
    st = dict(inp)
    model.forward_static(st, capacity=M_FINE)
    assert st["b_ids"].shape[0] == M_FINE and 2 * M_FINE * 25 * 256 > 2 ** 31
    util.assert_static_equals_eager(st, eager, "forward_static capacity past 2^31")
    _record("forward_static_2_31", peak, matches=int(eager["b_ids"].shape[0]))
