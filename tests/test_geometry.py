"""Robust two-view geometry (`loftr_b200.estimate_geometry`, `match_features(..., estimate=...)`).

tests/geometry_ref.py carries a float64 NumPy implementation of the same estimator (sample draw, minimal solvers,
errors, MSAC ranking, refit).  The GPU runs the geometry in fp64 too, so on identical samples the winning hypothesis
must agree exactly and the refitted model to rounding.  Synthetic scenes with known H / F check accuracy; the CPU tests
check the reference, its mirror of the library's workspace and the host-side validation, and run without a GPU.
tests/test_geometry_edges_gpu.py checks the kernels' intermediate results at their launch boundaries."""
import numpy as np
import pytest
import torch

import loftr_b200
from geometry_ref import (S, STAGE, STAGING_THR, draw_samples, errors, model_dist, pad_batch, philox4x32_10, project_h,
                          ransac_ref, scene, solve_f8, solve_h4, staging_case, tile_ranking, ws_layout)
from loftr_b200 import geometry

DEV = "cuda:0"


def gpu(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in arrays]


# ---------------------------------------------------------------------------------------------- CPU tests
def test_philox_known_answer():
    # Random123 known-answer vector for philox4x32_10 with zero counter and key
    got = philox4x32_10(np.zeros((1, 4), np.uint32), (0, 0))[0]
    assert [hex(int(v)) for v in got] == ["0x6627e8d5", "0xe169c58d", "0xbc57ac4c", "0x9b00dbd8"]


def test_draw_samples_distinct_sorted_and_covering():
    for n, s in ((4, 4), (8, 8), (9, 8), (1000, 4)):
        smp = draw_samples(5, 3, n, s, 300)
        assert smp.min() >= 0 and smp.max() < n
        assert (np.diff(smp, axis=1) > 0).all()
    # K == s: every hypothesis draws the whole set
    assert (draw_samples(0, 0, 4, 4, 20) == np.arange(4)).all()
    smp = draw_samples(1, 0, 10, 4, 4000)
    assert len(np.unique(smp)) == 10 and abs(np.bincount(smp.ravel()).std() / 1600) < 0.1


@pytest.mark.parametrize("model", ["homography", "fundamental"])
def test_reference_recovers_synthetic_model(model):
    rs = np.random.RandomState(3)
    p0, p1, inl, gt, _ = scene(rs, model, 300, 0.3)
    r = ransac_ref(p0, p1, model, 3.0, 512 if model == "homography" else 2048)
    assert model_dist(r["model"], gt) < 0.02
    assert (r["mask"] & inl).sum() / inl.sum() > 0.97 and (r["mask"] & inl).sum() / r["mask"].sum() > 0.95


def test_reference_minimal_solvers_are_exact():
    rs = np.random.RandomState(0)
    p0, p1, _, gt, (c0, c1) = scene(rs, "homography", 4, 0.0, sigma=0.0)
    h, ok = solve_h4(p0[None].astype(np.float64), p1[None].astype(np.float64))
    assert ok[0] and model_dist(h[0], gt) < 1e-5
    p0, p1, _, gt, _ = scene(rs, "fundamental", 8, 0.0, sigma=0.0)
    f, ok = solve_f8(p0[None].astype(np.float64), p1[None].astype(np.float64))
    assert ok[0] and model_dist(f[0], gt) < 1e-3 and abs(np.linalg.det(f[0] / np.linalg.norm(f[0]))) < 1e-12


def test_reference_collinear_is_degenerate():
    t = np.linspace(0, 1, 50)
    p0 = np.stack([10 + 500 * t, 20 + 300 * t], 1).astype(np.float32)
    for model in S:
        r = ransac_ref(p0, p0 + 5, model, 2.0, 64)
        assert r["best"] == -1 and np.isnan(r["model"]).all() and r["count"] == 0


def test_host_validation_without_gpu():
    cpu = torch.zeros(2, 16, 2)
    with pytest.raises(ValueError, match="CUDA"):
        loftr_b200.estimate_geometry(cpu, cpu)
    with pytest.raises(TypeError, match="float32"):
        loftr_b200.estimate_geometry(cpu.double(), cpu.double())
    with pytest.raises(ValueError, match="model"):
        loftr_b200.estimate_geometry(cpu, cpu, model="essential")
    for bad in (0, -1.0, float("nan"), float("inf"), True):
        with pytest.raises(ValueError, match="threshold"):
            geometry.check_options(threshold=bad)
    for bad in (0, 2 ** 31, 1.5):
        with pytest.raises(ValueError, match="iterations"):
            geometry.check_options(iterations=bad)
    with pytest.raises(ValueError, match="seed"):
        geometry.check_options(seed=-1)


def test_workspace_layout_mirror_matches_the_library():
    """ws_layout (how tests/test_geometry_edges_gpu.py reads the kernels' intermediate results back) is the library's
    geometry_ws_layout; the size query needs no device."""
    from loftr_b200 import _lib
    lib = _lib.load()
    for B in (0, 1, 3, 65535):
        for K in (4, 8, 255, 257, 19200):
            for it in (1, 63, 64, 65, 129, 2048):
                assert lib.lb_geometry_workspace_bytes(B, K, it) == ws_layout(B, K, it)["total"], (B, K, it)
    lay = ws_layout(3, 5, 65)
    assert (lay["compact_col"], lay["n_valid"], lay["tile_best"], lay["n_tiles"]) == (240, 304, 320, 2)


@pytest.mark.parametrize("model", list(S))
def test_staging_cases_bite_on_the_reference(model):
    """The staging grid of test_geometry_edges_gpu.py would catch a scoring loop that stops after its first round of
    STAGE matches (another winner from n = 2048 on) or skips a partial last round (another tile count whenever one
    exists: at n = 1025 the lone match of round 2 is an inlier)."""
    for n in (1025, 2048, 2049, 4100):
        p0, p1, it, seed = staging_case(model, n)
        full = tile_ranking(p0, p1, model, STAGING_THR, it, seed)
        win = lambda r: r[2][np.lexsort((r[2], r[1], -r[0]))[0]]
        if n >= 2 * STAGE:
            assert win(full) != win(tile_ranking(p0, p1, model, STAGING_THR, it, seed, upto=STAGE)), n
        if n % STAGE:
            partial = tile_ranking(p0, p1, model, STAGING_THR, it, seed, upto=n - n % STAGE)
            assert (partial[0] != full[0]).any(), n


# ---------------------------------------------------------------------------------------------- GPU tests
def _run(P0, P1, V, model, thr=3.0, iterations=1024, seed=0, details=True, **kw):
    p0, p1, v = gpu(P0, P1, V)
    out = loftr_b200.estimate_geometry(p0, p1, v, model=model, threshold=thr, iterations=iterations, seed=seed,
                                       return_details=details, **kw)
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["homography", "fundamental"])
def test_matches_numpy_reference_hypothesis_for_hypothesis(model):
    rs = np.random.RandomState(11)
    ns = [300, 9, 120, 1000, 57]
    pairs = [scene(rs, model, n, r)[:2] for n, r in zip(ns, [0.3, 0.0, 0.5, 0.2, 0.4])]
    P0, P1, V, cols = pad_batch(pairs, 1100, rs)
    iters, seed = 700, 12345678901
    H, mask, cnt, det = _run(P0, P1, V, model, 2.5, iters, seed)
    H, mask, cnt = H.cpu().numpy(), mask.cpu().numpy(), cnt.cpu().numpy()
    best, samples = det["best_hypothesis"].cpu().numpy(), det["samples"].cpu().numpy()
    for b, (a, c) in enumerate(pairs):
        ref = ransac_ref(a, c, model, 2.5, iters, seed, b)
        assert (samples[b] == cols[b][ref["samples"]]).all(), b
        assert best[b] == ref["best"], b
        assert cnt[b] == ref["count"], b
        assert (np.flatnonzero(mask[b]) == cols[b][ref["mask"]]).all(), b
        assert not mask[b][~V[b]].any()
        assert model_dist(H[b], ref["model"]) < 2e-6, (b, H[b], ref["model"])
        np.testing.assert_allclose(H[b], ref["model"], rtol=1e-5, atol=1e-5 * np.abs(ref["model"]).max())


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["homography", "fundamental"])
@pytest.mark.parametrize("outliers", [0.0, 0.3, 0.6])
def test_ground_truth_accuracy(model, outliers):
    rs = np.random.RandomState(int(outliers * 10) + (0 if model == "homography" else 50))
    ns = [800, 200, 2048, 500, 64, 1500]
    scenes = [scene(rs, model, n, outliers) for n in ns]
    P0, P1, V, cols = pad_batch([sc[:2] for sc in scenes], 2048, rs)
    iters = 2048 if model == "homography" or outliers < 0.5 else 16384
    M, mask, cnt = _run(P0, P1, V, model, 3.0, iters, 7, details=False)
    M, mask, cnt = M.cpu().numpy(), mask.cpu().numpy(), cnt.cpu().numpy()
    for b, (p0, p1, inl, gt, (c0, c1)) in enumerate(scenes):
        assert np.isfinite(M[b]).all()
        assert not mask[b][~V[b]].any()
        got = mask[b][cols[b]]
        assert cnt[b] == got.sum()
        tp = (got & inl).sum()
        assert tp / inl.sum() > 0.95 and tp / got.sum() > 0.95, (b, tp, inl.sum(), got.sum())
        if model == "homography":
            grid = np.stack(np.meshgrid(np.linspace(0, 640, 9), np.linspace(0, 480, 7)), -1).reshape(-1, 2)
            err = np.linalg.norm(project_h(M[b].astype(np.float64), grid) - project_h(gt, grid), axis=1)
            # bounded by extrapolation to the image corners from the fewest inliers (80 of 200 at 60 % outliers)
            assert err.max() < 4.0 and err.mean() < 1.0, (b, err.max(), err.mean())
            assert abs(M[b, 2, 2] - 1) < 1e-6
        else:
            e = np.sqrt(errors("fundamental", M[b].astype(np.float64), c0, c1))
            assert np.median(e) < 0.5 and np.mean(e) < 1.0, (b, np.median(e))
            assert abs(np.linalg.norm(M[b]) - 1) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["homography", "fundamental"])
def test_degenerate_and_small_pairs(model):
    s = S[model]
    rs = np.random.RandomState(2)
    t = rs.uniform(0, 1, 100)
    line = np.stack([10 + 600 * t, 30 + 400 * t], 1).astype(np.float32)
    good = scene(rs, model, 200, 0.2)[:2]
    exact = scene(rs, model, s, 0.0, sigma=0.0)[:2]
    pairs = [(line, line * 0.5 + 20), good, (good[0][:s - 1], good[1][:s - 1]), (good[0][:0], good[1][:0]), exact]
    P0, P1, V, cols = pad_batch(pairs, 256)
    M, mask, cnt, det = _run(P0, P1, V, model, 2.0, 256)
    M, mask, cnt, best = M.cpu().numpy(), mask.cpu().numpy(), cnt.cpu().numpy(), det["best_hypothesis"].cpu().numpy()
    for b in (0, 2, 3):    # collinear, below the sample size, empty: NaN model, nothing marked
        assert np.isnan(M[b]).all() and cnt[b] == 0 and not mask[b].any() and best[b] == -1, b
    assert (det["samples"][2:4].cpu().numpy() == -1).all()
    for b in (1, 4):
        assert np.isfinite(M[b]).all() and cnt[b] >= s and best[b] >= 0
    assert cnt[4] == s
    # K equal to the sample size, B = 1
    M1, mask1, cnt1 = _run(P0[4:5, :s], P1[4:5, :s], V[4:5, :s], model, 2.0, 64, details=False)
    assert cnt1.item() == s and mask1.all() and torch.isfinite(M1).all()
    # K below the sample size is refused before any launch
    with pytest.raises(ValueError, match="sample size"):
        _run(P0[:, :s - 1], P1[:, :s - 1], V[:, :s - 1], model)


@pytest.mark.gpu
def test_large_batch_and_count_form_of_valid():
    rs = np.random.RandomState(5)
    B, K = 3000, 96
    pairs = [scene(rs, "homography", int(n), 0.25)[:2] for n in rs.randint(0, K + 1, B)]
    P0, P1, V, _ = pad_batch(pairs, K)
    M, mask, cnt = _run(P0, P1, V, "homography", 3.0, 256, details=False)
    counts = torch.tensor([len(a) for a, _ in pairs], device=DEV)
    p0, p1 = gpu(P0, P1)
    M2, mask2, cnt2 = loftr_b200.estimate_geometry(p0, p1, counts, iterations=256)
    assert torch.equal(M.nan_to_num(7.0), M2.nan_to_num(7.0)) and torch.equal(mask, mask2) and torch.equal(cnt, cnt2)
    ok = counts >= 4
    assert torch.isnan(M[~ok]).all() and (cnt[~ok] == 0).all()
    assert torch.isfinite(M[ok & (cnt > 0)]).all()
    assert not mask[~torch.from_numpy(V).to(DEV)].any()


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["homography", "fundamental"])
def test_deterministic_and_independent_of_batch_composition(model):
    rs = np.random.RandomState(9)
    pairs = [scene(rs, model, n, 0.4)[:2] for n in (400, 150, 600, 90)]
    P0, P1, V, cols = pad_batch(pairs, 640, rs)
    a = _run(P0, P1, V, model, 3.0, 512, 3, details=False)
    b = _run(P0, P1, V, model, 3.0, 512, 3, details=False)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # pairs 2 and 0 alone, in another order, packed at the front of a different K, keyed by their ids
    Q0, Q1, QV, qcols = pad_batch([pairs[2], pairs[0]], 700)
    ids = torch.tensor([2, 0], device=DEV)
    c = _run(Q0, Q1, QV, model, 3.0, 512, 3, details=False, pair_ids=ids)
    for qb, b_ in ((0, 2), (1, 0)):
        assert torch.equal(c[0][qb], a[0][b_]) and torch.equal(c[2][qb], a[2][b_])
        assert torch.equal(c[1][qb][torch.from_numpy(qcols[qb]).to(DEV)], a[1][b_][torch.from_numpy(cols[b_]).to(DEV)])
    # a neighbour's data does not reach pair 1
    R0 = P0.copy()
    R0[0] = rs.uniform(0, 640, R0[0].shape)
    d = _run(R0, P1, V, model, 3.0, 512, 3, details=False)
    assert torch.equal(d[0][1:], a[0][1:]) and torch.equal(d[1][1:], a[1][1:]) and torch.equal(d[2][1:], a[2][1:])
    # another seed draws other samples
    e = _run(P0, P1, V, model, 3.0, 512, 4)
    assert not torch.equal(e[3]["samples"], _run(P0, P1, V, model, 3.0, 512, 3)[3]["samples"])


@pytest.mark.gpu
def test_cuda_graph_capture_and_replay():
    rs = np.random.RandomState(4)
    pairs = [scene(rs, "homography", n, 0.3)[:2] for n in (300, 500)]
    P0, P1, V, _ = pad_batch(pairs, 512)
    p0, p1, v = gpu(P0, P1, V)
    ref = loftr_b200.estimate_geometry(p0, p1, v, iterations=512)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        loftr_b200.estimate_geometry(p0, p1, v, iterations=512)   # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = loftr_b200.estimate_geometry(p0, p1, v, iterations=512)
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(out, ref):
        assert torch.equal(x, y)
    p1.copy_(p0)                     # new data in place: identity homography
    g.replay()
    torch.cuda.synchronize()
    assert torch.allclose(out[0], torch.eye(3, device=DEV).expand(2, 3, 3), atol=1e-4)
    assert torch.equal(out[2].cpu(), torch.tensor([300, 500], dtype=torch.int32))


def _model():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    import weights as W
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict({k: torch.from_numpy(v) for k, v in W.make_state(shapes, seed=0).items()})
    return model.to(DEV)


def _warped_pair(h_true, hw=(240, 320), seed=0):
    """A textured image and its warp by h_true (image1(x1) = image0(h_true^-1 x1)) via grid_sample."""
    g = torch.Generator().manual_seed(seed)
    hh, ww = hw
    img = torch.nn.functional.interpolate(torch.rand(1, 1, hh // 4, ww // 4, generator=g), size=hw, mode="bicubic",
                                          align_corners=False).clamp(0, 1)
    ys, xs = torch.meshgrid(torch.arange(hh, dtype=torch.float64), torch.arange(ww, dtype=torch.float64),
                            indexing="ij")
    pts = torch.stack([xs, ys, torch.ones_like(xs)], -1) @ torch.from_numpy(np.linalg.inv(h_true)).T
    src = pts[..., :2] / pts[..., 2:]
    grid = torch.stack([(src[..., 0] + 0.5) / ww * 2 - 1, (src[..., 1] + 0.5) / hh * 2 - 1], -1)[None].float()
    warped = torch.nn.functional.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
    return img, warped


@pytest.mark.gpu
def test_match_features_estimate_flag_on_a_warped_pair():
    """A textured image and its warp by a known homography.  The flag leaves every key of the plain call bit for bit
    and adds a model that explains the inliers it marks.  The test weights are random, so the matches follow the
    position encoding more than the image content, and the true H is not what they support: the accuracy of the
    estimator against a known model is covered on synthetic matches above."""
    model = _model()
    h_true = np.array([[1.0, 0.0, 16.0], [0.0, 1.0, 8.0], [0.0, 0.0, 1.0]])
    img0, img1 = _warped_pair(h_true)
    bank = model.extract_features(torch.cat([img0, img1]).to(DEV))
    i0, i1 = torch.tensor([0], device=DEV), torch.tensor([1], device=DEV)
    plain = model.match_features(bank, i0, bank, i1)
    again = model.match_features(bank, i0, bank, i1, estimate=None)
    assert set(again) == set(plain) and all(torch.equal(plain[k], again[k]) for k in plain if torch.is_tensor(plain[k]))
    got = model.match_features(bank, i0, bank, i1, estimate={"model": "homography", "threshold": 2.0})
    assert set(got) == set(plain) | {"geom_model", "geom_inliers", "geom_num_inliers"}
    for k in plain:
        if torch.is_tensor(plain[k]):
            assert torch.equal(plain[k], got[k]), k
    assert got["geom_inliers"].shape == plain["m_bids"].shape and got["geom_model"].shape == (1, 3, 3)
    n_in = int(got["geom_num_inliers"][0])
    assert n_in == int(got["geom_inliers"].sum()) >= 8
    H = got["geom_model"][0].double().cpu().numpy()
    inl = got["geom_inliers"].cpu().numpy()
    e = errors("homography", H, got["mkpts0_f"].double().cpu().numpy()[inl], got["mkpts1_f"].double().cpu().numpy()[inl])
    assert np.sqrt(e).max() < 2.0 + 1e-3


@pytest.mark.gpu
def test_match_features_estimate_is_the_estimator_on_the_padded_list():
    model = _model()
    h_true = np.array([[1.02, 0.03, 10.0], [-0.02, 0.99, 12.0], [1e-5, 0.0, 1.0]])
    imgs = [_warped_pair(h_true, seed=s) for s in (1, 2)]
    bank = model.extract_features(torch.cat([im for pair in imgs for im in pair]).to(DEV))
    i0, i1 = torch.tensor([0, 2], device=DEV), torch.tensor([1, 3], device=DEV)
    opts = {"model": "fundamental", "threshold": 1.5, "iterations": 1024, "seed": 5}
    out = model.match_features(bank, i0, bank, i1, estimate=opts)
    bids = out["m_bids"].cpu().numpy()
    pairs = [(out["mkpts0_f"].cpu().numpy()[bids == b], out["mkpts1_f"].cpu().numpy()[bids == b]) for b in range(2)]
    P0, P1, V, _ = pad_batch(pairs, max(8, max(len(a) for a, _ in pairs)))
    M, mask, cnt = _run(P0, P1, V, "fundamental", 1.5, 1024, 5, details=False)
    assert torch.equal(out["geom_model"].nan_to_num(3.0), M.nan_to_num(3.0)) and torch.equal(out["geom_num_inliers"], cnt)
    assert torch.equal(out["geom_inliers"], mask[torch.from_numpy(V).to(DEV)])
    with pytest.raises(ValueError, match="estimate"):
        model.match_features(bank, i0, bank, i1, estimate={"model": "homography", "bogus": 1})
