"""The geometry estimator's three kernels against the float64 reference of tests/geometry_ref.py, at their launch
boundaries, from the kernels' own intermediate results.

lb_estimate_geometry runs here into a workspace the test allocates (ws_layout mirrors geometry_ws_layout), so besides
the final model, mask and count the test reads back what geometry_compact_kernel stored (compact, compact_col,
n_valid) and every scoring tile's winner (tile_best: count, MSAC cost, hypothesis index).  Each grid point names the
branch it covers:

- staging rounds of geometry_score_kernel (kGeoStage = 1024 matches per round): n = 1023, 1024, 1025 (a lone match in
  round 2, an inlier), 2048, 2049 (a 1-match third round), 4100 and the matcher's largest per-pair count 19200 (19
  rounds).  From n = 2048 on, round 1 holds a weak structure and the dominant one follows it, so a scoring loop that
  stopped after round 1 would rank another winner (tests/test_geometry.py asserts that on the reference);
- hypothesis tiles (kGeoHypPerBlock = 64): 1, 63, 64, 65 and 129 iterations;
- geometry_compact_kernel's 256-column chunks: K = 255, 256, 257, 513;
- geometry_refit_kernel's 256-thread strides and block sums: 255, 256 and 257 final inliers;
- exact ties: n == s (every hypothesis draws the same sample) and n == s + 1;
- the RNG key: pair ids 0, 2**31 - 1, -1 and 2**32 + 3 (int64) with seed 2**64 - 1;
- the grid-y limit B = 65535 (and B = 65536 refused before any launch);
- NaN and +-inf coordinates in valid slots.

Counts and indices must match exactly.  Costs match to cost_rtol (1e-12, wider for an ill-conditioned 8-point sample)
plus an absolute 1e-20 px^2 per match.  Where the reference's best two costs in a tile are closer than 1e-9 relative
(or than those tolerances), either winner is accepted and counted in the record of the grid point."""
import ctypes as C

import numpy as np
import pytest
import torch

import geometry_ref as G
import util
import loftr_b200
from loftr_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODELS = list(G.S)
NEAR_TIE = 1e-9
# absolute floor of a cost comparison per match, in px^2: a transfer residual of 1e-10 px, the rounding level of a
# sample the model fits exactly (n == s: every error is ~1e-25 and so is the cost)
COST_ATOL = 1e-20


def run(P0, P1, V, model, thr, iterations, seed=0, pair_ids=None):
    """lb_estimate_geometry through ctypes with a workspace of our own -> outputs plus the decoded workspace."""
    B, K = P0.shape[:2]
    s = G.S[model]
    lay = G.ws_layout(B, K, iterations)
    lib = _lib.load()
    assert lib.lb_geometry_workspace_bytes(B, K, iterations) == lay["total"]
    p0, p1 = (torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV) for a in (P0, P1))
    v = None if V is None else torch.from_numpy(np.ascontiguousarray(V, np.uint8)).to(DEV)
    ids = None if pair_ids is None else torch.as_tensor(pair_ids, dtype=torch.int32, device=DEV)
    ws = torch.full((lay["total"],), 0xA5, dtype=torch.uint8, device=DEV)
    mdl = torch.empty(B, 3, 3, device=DEV)
    mask = torch.empty(B, K, dtype=torch.uint8, device=DEV)
    cnt = torch.empty(B, dtype=torch.int32, device=DEV)
    best = torch.empty(B, dtype=torch.int32, device=DEV)
    smp = torch.empty(B, iterations, s, dtype=torch.int32, device=DEV)
    _lib.check(lib.lb_estimate_geometry(p0.data_ptr(), p1.data_ptr(), _lib.ptr(v), _lib.ptr(ids), B, K,
                                        _lib.GEOMETRY_HOMOGRAPHY if model == "homography" else _lib.GEOMETRY_FUNDAMENTAL,
                                        thr, iterations, seed, mdl.data_ptr(), mask.data_ptr(), cnt.data_ptr(),
                                        best.data_ptr(), smp.data_ptr(), ws.data_ptr(), lay["total"],
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    w = ws.cpu().numpy()
    region = lambda name, nbytes: w[lay[name]:lay[name] + nbytes]
    return {"model": mdl.cpu().numpy(), "mask": mask.cpu().numpy().astype(bool), "count": cnt.cpu().numpy(),
            "best": best.cpu().numpy(), "samples": smp.cpu().numpy(),
            "compact": region("compact", B * K * 16).view(np.float32).reshape(B, K, 4),
            "compact_col": region("compact_col", B * K * 4).view(np.int32).reshape(B, K),
            "n_valid": region("n_valid", B * 4).view(np.int32),
            "tiles": region("tile_best", B * lay["n_tiles"] * 16).view(G.GEO_BEST).reshape(B, lay["n_tiles"])}


def check_compaction(out, b, P0, P1, V):
    cols = np.flatnonzero(V[b]) if V is not None else np.arange(P0.shape[1])
    n = len(cols)
    assert out["n_valid"][b] == n, (b, out["n_valid"][b], n)
    want = np.concatenate([P0[b, cols], P1[b, cols]], 1).astype(np.float32)
    assert np.array_equal(out["compact"][b, :n].view(np.uint32), want.view(np.uint32)), b
    assert np.array_equal(out["compact_col"][b, :n], cols), b
    return cols


def check_tiles(out, b, p0, p1, model, thr, iterations, seed, pair_id, cols):
    """Every tile winner of pair b against tile_ranking -> stats; near-ties adjudicated."""
    cnt, cost, hyp, h = G.tile_ranking(p0, p1, model, thr, iterations, seed, pair_id)
    if h is not None:
        h["n"] = len(p0)
    got = out["tiles"][b]
    assert len(got) == len(hyp)
    ties, worst = 0, 0.0
    for t, g in enumerate(got):
        if cnt[t] < 0:      # every hypothesis of the tile degenerate (or the pair below the sample size)
            assert (g["count"], g["sum"], g["hyp"]) == (-1, 0.0, t * G.HYP_PER_TILE), (b, t, g)
            continue
        k = int(g["hyp"])
        assert t * G.HYP_PER_TILE <= k < min((t + 1) * G.HYP_PER_TILE, iterations), (b, t, k)
        if k != hyp[t]:
            assert near_tie(h, k, hyp[t]), (b, t, k, int(hyp[t]), int(h["count"][k]), int(cnt[t]))
            ties += 1
        assert g["count"] == h["count"][k], (b, t, k, int(g["count"]), int(h["count"][k]))
        tol = h["cost_rtol"][k] * h["cost"][k] + len(p0) * COST_ATOL
        assert abs(g["sum"] - h["cost"][k]) <= tol, (b, t, k, g["sum"], h["cost"][k], h["cost_rtol"][k])
        worst = max(worst, abs(g["sum"] - h["cost"][k]) / tol)
    if h is not None:
        assert np.array_equal(out["samples"][b], cols[h["samples"]]), b
    return {"tiles": len(got), "tiles_equal": int((got["hyp"] == hyp).sum()), "near_ties": ties,
            "max_cost_err_over_tol": worst}, h


def near_tie(h, a, b):
    """Hypotheses a and b have the same count and costs the reference cannot order."""
    tol = max(NEAR_TIE, h["cost_rtol"][a] + h["cost_rtol"][b]) * h["cost"][b] + 2 * h["n"] * COST_ATOL
    return h["count"][a] == h["count"][b] and abs(h["cost"][a] - h["cost"][b]) < tol


def check_final(out, b, p0, p1, model, thr, iterations, seed, pair_id, cols, stats, h):
    ref = G.ransac_ref(p0, p1, model, thr, iterations, seed, pair_id)
    best = out["best"][b]
    if best != ref["best"]:      # only a near-tie may move the winner, and then the refit starts elsewhere
        assert best >= 0 and ref["best"] >= 0 and near_tie(h, best, ref["best"]), (b, best, ref["best"])
        stats["near_ties"] += 1
        return
    assert out["count"][b] == ref["count"], (b, out["count"][b], ref["count"])
    assert np.array_equal(np.flatnonzero(out["mask"][b]), cols[ref["mask"]]), b
    if ref["best"] < 0:
        assert np.isnan(out["model"][b]).all()
        return
    assert model_dist_ok(out["model"][b], ref["model"]), (b, out["model"][b], ref["model"])


def model_dist_ok(got, ref):
    return G.model_dist(got, ref) < 2e-6 and np.allclose(got, ref, rtol=1e-5, atol=1e-5 * np.abs(ref).max())


def check_pair(out, b, P0, P1, V, model, thr, iterations, seed=0, pair_id=None):
    cols = check_compaction(out, b, P0, P1, V)
    p0, p1 = P0[b, cols], P1[b, cols]
    pid = b if pair_id is None else pair_id
    stats, h = check_tiles(out, b, p0, p1, model, thr, iterations, seed, pid, cols)
    check_final(out, b, p0, p1, model, thr, iterations, seed, pid, cols, stats, h)
    assert not out["mask"][b][np.setdiff1d(np.arange(P0.shape[1]), cols)].any()
    return stats, h


# ---------------------------------------------------------------------------------------------- staging rounds
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("n", G.STAGING_N)
def test_scoring_rounds(n, model):
    p0, p1, iterations, seed = G.staging_case(model, n)
    K = n if n == 19200 else n + 61
    rs = np.random.RandomState(n)
    P0, P1, V, _ = G.pad_batch([(p0, p1)], K, rs)
    out = run(P0, P1, V, model, G.STAGING_THR, iterations, seed)
    stats, _ = check_pair(out, 0, P0, P1, V, model, G.STAGING_THR, iterations, seed)
    util.record(f"geometry_rounds_{model}_n{n}", {"rounds": -(-n // G.STAGE), **stats})


# ---------------------------------------------------------------------------------------------- hypothesis tiles
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("iterations", [1, 63, 64, 65, 129])
def test_hypothesis_tiles(iterations, model):
    rs = np.random.RandomState(iterations)
    pairs = [G.scene(rs, model, n, 0.3)[:2] for n in (300, 41)]
    P0, P1, V, _ = G.pad_batch(pairs, 320, rs)
    out = run(P0, P1, V, model, 3.0, iterations, 77)
    stats = [check_pair(out, b, P0, P1, V, model, 3.0, iterations, 77)[0] for b in range(2)]
    util.record(f"geometry_tiles_{model}_it{iterations}", {k: sum(s[k] for s in stats) for k in stats[0]})


# ---------------------------------------------------------------------------------------------- compaction chunks
@pytest.mark.parametrize("K", [255, 256, 257, 513])
def test_compaction_chunks(K):
    """Model-independent: one model runs it.  Rows: entries on both sides of every 256-column chunk edge among random
    ones, all valid, none valid, only column K - 1, and prefixes (the count form of `valid`)."""
    rs = np.random.RandomState(K)
    rows = []
    edge = rs.rand(K) < 0.5
    for c in range(256, K + 1, 256):
        edge[c - 1] = True
        if c < K:
            edge[c] = True
    last = np.zeros(K, bool)
    last[K - 1] = True
    counts = [K, 1, min(256, K), K // 2 + 1, 0]
    rows = [edge, np.ones(K, bool), np.zeros(K, bool), last] + [np.arange(K) < c for c in counts]
    V = np.stack(rows)
    B = len(rows)
    P0 = rs.uniform(0, 640, (B, K, 2)).astype(np.float32)
    P1 = (P0 + rs.normal(0, 2, P0.shape)).astype(np.float32)
    out = run(P0, P1, V, "homography", 3.0, 64, 5)
    for b in range(B):
        check_compaction(out, b, P0, P1, V)
    # the count form of `valid` is the prefix mask (the prefix rows keyed by their ids in the call above)
    tail = slice(4, B)
    p0, p1 = (torch.from_numpy(a[tail]).to(DEV) for a in (P0, P1))
    ids = torch.arange(4, B, device=DEV)
    a = loftr_b200.estimate_geometry(p0, p1, torch.tensor(counts, device=DEV), iterations=64, seed=5, pair_ids=ids)
    m = loftr_b200.estimate_geometry(p0, p1, torch.from_numpy(V[tail]).to(DEV), iterations=64, seed=5, pair_ids=ids)
    for x, y in zip(a, m):
        assert torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))
    assert np.array_equal(a[1].cpu().numpy(), out["mask"][tail]) and np.array_equal(a[2].cpu().numpy(), out["count"][tail])
    util.record(f"geometry_compaction_K{K}", {"rows": B, "n_valid": [int(x) for x in out["n_valid"]]})


# ---------------------------------------------------------------------------------------------- refit strides
def exact_scene(rs, model, n_in, n_out, thr, iterations, seed, sigma=0.3):
    """n_in inliers of one model and n_out outliers, shuffled, such that the reference's final mask is exactly the
    inliers: an outlier the estimate would count is drawn again."""
    p0, p1 = G.scene(rs, model, n_in + n_out, 0.0, sigma)[:2]
    out = rs.permutation(n_in + n_out)[:n_out]
    for _ in range(20):
        extra = out[G.ransac_ref(p0, p1, model, thr, iterations, seed)["mask"][out]]
        if len(extra) == 0:
            break
        p1[extra] = rs.uniform((0, 0), (640, 480), (len(extra), 2))
    return p0, p1


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("outliers", [0, 100])
@pytest.mark.parametrize("inliers", [255, 256, 257])
def test_refit_strides(inliers, outliers, model):
    rs = np.random.RandomState(inliers + outliers)
    iterations = 128 if model == "homography" else 512
    p0, p1 = exact_scene(rs, model, inliers, outliers, 3.0, iterations, 9)
    P0, P1, V, _ = G.pad_batch([(p0, p1)], inliers + outliers + 3, rs)
    out = run(P0, P1, V, model, 3.0, iterations, 9)
    assert G.ransac_ref(p0, p1, model, 3.0, iterations, 9)["count"] == inliers   # the case reaches its count
    stats, _ = check_pair(out, 0, P0, P1, V, model, 3.0, iterations, 9)
    assert out["count"][0] == inliers
    util.record(f"geometry_refit_{model}_in{inliers}_out{outliers}", stats)


# ---------------------------------------------------------------------------------------------- exact ties
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("extra", [0, 1])
def test_exact_ties(extra, model):
    s = G.S[model]
    rs = np.random.RandomState(40 + extra)
    p0, p1 = G.scene(rs, model, s + extra, 0.0, 0.5)[:2]
    P0, P1, V, _ = G.pad_batch([(p0, p1)], s + extra + 2, rs)
    iterations = 200
    out = run(P0, P1, V, model, 3.0, iterations, 3)
    stats, h = check_pair(out, 0, P0, P1, V, model, 3.0, iterations, 3)
    tiles = out["tiles"][0]
    smp = out["samples"][0]
    for t, g in enumerate(tiles):
        lo = t * G.HYP_PER_TILE
        same = [k for k in range(lo, min(lo + G.HYP_PER_TILE, iterations)) if np.array_equal(smp[k], smp[g["hyp"]])]
        assert g["hyp"] == same[0], (t, int(g["hyp"]), same[:3])   # the smallest index among identical samples
    if extra == 0:
        assert out["best"][0] == 0 and list(tiles["hyp"]) == [t * G.HYP_PER_TILE for t in range(len(tiles))]
        assert stats["near_ties"] == 0
    util.record(f"geometry_ties_{model}_n{s + extra}", stats)


# ---------------------------------------------------------------------------------------------- RNG key
@pytest.mark.parametrize("model", MODELS)
def test_pair_ids_key_modulo_2_32(model):
    rs = np.random.RandomState(12)
    ids = [0, 2 ** 31 - 1, -1, 2 ** 32 + 3]
    pairs = [G.scene(rs, model, n, 0.3)[:2] for n in (200, 150, 90, 240)]
    P0, P1, V, cols = G.pad_batch(pairs, 256, rs)
    seed, iterations = 2 ** 64 - 1, 192
    p0, p1, v = (torch.from_numpy(a).to(DEV) for a in (P0, P1, V))
    got = loftr_b200.estimate_geometry(p0, p1, v, model=model, iterations=iterations, seed=seed,
                                       pair_ids=torch.tensor(ids, dtype=torch.int64, device=DEV), return_details=True)
    ids32 = [(i + 2 ** 31) % 2 ** 32 - 2 ** 31 for i in ids]     # the same ids as int32
    narrow = loftr_b200.estimate_geometry(p0, p1, v, model=model, iterations=iterations, seed=seed,
                                          pair_ids=torch.tensor(ids32, dtype=torch.int32, device=DEV))
    for x, y in zip(got[:3], narrow):
        assert torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))
    out = run(P0, P1, V, model, 3.0, iterations, seed, ids32)
    stats = []
    for b, pid in enumerate(ids):
        st, _ = check_pair(out, b, P0, P1, V, model, 3.0, iterations, seed, pid % 2 ** 32)
        stats.append(st)
        ref = G.ransac_ref(*pairs[b], model, 3.0, iterations, seed, pid % 2 ** 32)
        assert np.array_equal(got[3]["samples"][b].cpu().numpy(), cols[b][ref["samples"]]), pid
        assert got[3]["best_hypothesis"][b].item() == out["best"][b] and got[2][b].item() == out["count"][b]
    util.record(f"geometry_pair_ids_{model}", {k: sum(s[k] for s in stats) for k in ("tiles", "tiles_equal",
                                                                                  "near_ties")})


# ---------------------------------------------------------------------------------------------- grid-y limit
@pytest.mark.parametrize("model", MODELS)
def test_grid_y_limit(model):
    """B = 65535 pairs of K = s matches (H: K = 4) in one call; the score kernel's grid is (1, 65535)."""
    s = G.S[model]
    B, K, iterations = 65535, s, 64
    rs = np.random.RandomState(65535 + s)
    P0 = rs.uniform(0, 640, (B, K, 2)).astype(np.float32)
    P1 = (P0 * rs.uniform(0.9, 1.1, (B, 1, 1)) + rs.uniform(-20, 20, (B, 1, 2)) + rs.normal(0, 1, (B, K, 2)))
    P1 = P1.astype(np.float32)
    V = np.ones((B, K), bool)
    V[rs.rand(B) < 0.1, 0] = False            # a tenth of the rows below the sample size
    out = run(P0, P1, V, model, 3.0, iterations, 21)
    assert np.array_equal(out["n_valid"], V.sum(1))
    full = V.all(1)
    # n == s: every hypothesis draws the whole set, so the winner is hypothesis 0 or nothing
    assert set(np.unique(out["best"][full])) <= {0, -1} and (out["best"][~full] == -1).all()
    assert np.array_equal(out["best"] == 0, out["tiles"][:, 0]["count"] >= 0)
    rows = [0, 1, 32767, 40000 + int(np.flatnonzero(~full[40000:])[0]), B - 2, B - 1]
    for b in rows:
        p0, p1, v = (torch.from_numpy(a[b:b + 1]).to(DEV) for a in (P0, P1, V))
        alone = loftr_b200.estimate_geometry(p0, p1, v, model=model, iterations=iterations, seed=21,
                                             pair_ids=torch.tensor([b], device=DEV), return_details=True)
        assert torch.equal(alone[0][0].cpu().nan_to_num(7.0), torch.from_numpy(out["model"][b]).nan_to_num(7.0)), b
        assert np.array_equal(alone[1][0].cpu().numpy(), out["mask"][b]) and alone[2][0].item() == out["count"][b]
        assert alone[3]["best_hypothesis"][0].item() == out["best"][b]
    # one more pair is refused before any launch, by the package and by the C ABI
    p0, p1 = (torch.zeros(65536, K, 2, device=DEV) for _ in range(2))
    with pytest.raises(ValueError, match="65535"):
        loftr_b200.estimate_geometry(p0, p1, model=model)
    lib = _lib.load()
    launches = lib.lb_launch_count()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    rc = lib.lb_estimate_geometry(p0.data_ptr(), p1.data_ptr(), None, None, 65536, K, int(model == "fundamental"), 3.0,
                                  iterations, 0, ws.data_ptr(), ws.data_ptr(), ws.data_ptr(), None, None, ws.data_ptr(),
                                  ws.numel(), None)
    assert rc != 0 and b"65535" in lib.lb_last_error() and lib.lb_launch_count() == launches
    util.record(f"geometry_grid_y_{model}", {"B": B, "rows_checked": len(rows), "pairs_with_model": int((out["best"] == 0).sum())})


# ---------------------------------------------------------------------------------------------- non-finite input
@pytest.mark.parametrize("model", MODELS)
def test_non_finite_coordinates(model):
    rs = np.random.RandomState(31)
    p0, p1 = G.scene(rs, model, 300, 0.3)[:2]
    bad = rs.permutation(300)[:24]
    vals = [np.nan, np.inf, -np.inf]
    for i, k in enumerate(bad):
        (p0 if i % 2 else p1)[k, (i // 2) % 2] = vals[i % 3]
    p0[bad[-1]] = np.nan                       # both coordinates of one image
    P0, P1, V, cols = G.pad_batch([(p0, p1)], 333, rs)
    iterations = 256 if model == "homography" else 1024
    out = run(P0, P1, V, model, 3.0, iterations, 4)
    stats, h = check_pair(out, 0, P0, P1, V, model, 3.0, iterations, 4)
    bad_cols = set(cols[0][bad].tolist())
    assert not out["mask"][0][cols[0][bad]].any()
    assert out["best"][0] >= 0 and not bad_cols & set(out["samples"][0][out["best"][0]].tolist())
    for g in out["tiles"][0]:
        if g["count"] >= 0:
            assert not bad_cols & set(out["samples"][0][g["hyp"]].tolist())
    # a hypothesis drawing a non-finite slot is degenerate
    drew = np.isin(h["samples"], bad).any(1)
    assert drew.any() and (h["count"][drew] == -1).all()
    util.record(f"geometry_non_finite_{model}", {**stats, "hypotheses_on_non_finite": int(drew.sum())})
