"""Robust two-view geometry (`loftr_b200.estimate_geometry`, `match_features(..., estimate=...)`).

The file carries a float64 NumPy implementation of the same estimator: the same Philox4x32-10 sample draw, the same
minimal solvers (4-point normalised DLT with h33 = 1; normalised 8-point with rank 2), the same errors (symmetric
transfer, Sampson), the same MSAC ranking and the same Hartley-normalised least-squares refit.  The GPU runs the
geometry in fp64 too, so on identical samples the winning hypothesis must agree exactly and the refitted model to
rounding.  Synthetic scenes with known H / F check accuracy; the CPU tests check the reference and the host-side
validation and run without a GPU."""
import numpy as np
import pytest
import torch

import loftr_b200
from loftr_b200 import geometry

DEV = "cuda:0"
S = {"homography": 4, "fundamental": 8}


# ---------------------------------------------------------------------------------------------- NumPy reference
def philox4x32_10(ctr, key):
    """ctr [..., 4] uint32, key (k0, k1) -> [..., 4] uint32 (Random123's Philox4x32-10)."""
    c = [ctr[..., i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    m32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & m32
        k1 = (k1 + np.uint64(0xBB67AE85)) & m32
    return np.stack(c, -1).astype(np.uint32)


def draw_samples(seed, pair_id, n, s, iterations):
    """[iterations, s] ascending indices in [0, n): the kernel's draw (header of lb_estimate_geometry)."""
    hyp = np.arange(iterations, dtype=np.uint64)
    words = []
    for blk in range(2):
        ctr = np.stack([hyp, np.full_like(hyp, pair_id), np.full_like(hyp, blk), np.zeros_like(hyp)], -1)
        words.append(philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)))
    w = np.concatenate(words, -1).astype(np.uint64)
    out = np.empty((iterations, s), np.int64)
    for h in range(iterations):
        chosen = []
        for j in range(s):
            r = int((int(w[h, j]) * (n - j)) >> 32)
            for c in chosen:            # ascending
                if r >= c:
                    r += 1
            chosen.append(r)
            chosen.sort()
        out[h] = chosen
    return out


def norm_t(p):
    """Hartley normalisation [.., n, 2] -> (s, -s cx, -s cy) or None when the points coincide."""
    n = p.shape[-2]
    sx, sy = p[..., 0].sum(-1), p[..., 1].sum(-1)
    sq = (p ** 2).sum((-1, -2))
    cx, cy = sx / n, sy / n
    d2 = sq / n - (cx * cx + cy * cy)
    ok = d2 > 1e-24 * (sq / n) + 1e-300
    s = np.sqrt(2.0 / np.where(ok, d2, 1.0))
    return np.stack([s, -s * cx, -s * cy], -1), ok


def denormalise(model, mn, t0, t1):
    T0 = np.zeros(t0.shape[:-1] + (3, 3))
    T0[..., 0, 0] = T0[..., 1, 1] = t0[..., 0]
    T0[..., 0, 2], T0[..., 1, 2], T0[..., 2, 2] = t0[..., 1], t0[..., 2], 1
    T1 = np.zeros_like(T0)
    T1[..., 0, 0] = T1[..., 1, 1] = t1[..., 0]
    T1[..., 0, 2], T1[..., 1, 2], T1[..., 2, 2] = t1[..., 1], t1[..., 2], 1
    if model == "homography":
        return np.linalg.inv(T1) @ mn @ T0
    return np.swapaxes(T1, -1, -2) @ mn @ T0


def rank2(f):
    _, v = np.linalg.eigh(np.swapaxes(f, -1, -2) @ f)
    v0 = v[..., :, 0:1]
    return f - (f @ v0) @ np.swapaxes(v0, -1, -2)


def apply(t, p):
    return p * t[..., None, 0:1] + t[..., None, 1:3]


def solve_h4(p0, p1):
    """[..., 4, 2] -> (H [..., 3, 3], ok)."""
    t0, ok0 = norm_t(p0)
    t1, ok1 = norm_t(p1)
    u, u2 = apply(t0, p0), apply(t1, p1)
    ok = ok0 & ok1
    for q in (u, u2):
        for a, b, c in ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)):
            d1, d2 = q[..., b, :] - q[..., a, :], q[..., c, :] - q[..., a, :]
            ok &= np.abs(d1[..., 0] * d2[..., 1] - d1[..., 1] * d2[..., 0]) >= 1e-5
    A = np.zeros(p0.shape[:-2] + (8, 9))
    x, y, x2, y2 = u[..., 0], u[..., 1], u2[..., 0], u2[..., 1]
    A[..., 0::2, 0], A[..., 0::2, 1], A[..., 0::2, 2] = x, y, 1
    A[..., 0::2, 6], A[..., 0::2, 7], A[..., 0::2, 8] = -x * x2, -y * x2, x2
    A[..., 1::2, 3], A[..., 1::2, 4], A[..., 1::2, 5] = x, y, 1
    A[..., 1::2, 6], A[..., 1::2, 7], A[..., 1::2, 8] = -x * y2, -y * y2, y2
    idx = np.arange(A.shape[0])
    for c in range(8):                         # Gaussian elimination, partial pivoting (first maximum)
        piv = c + np.argmax(np.abs(A[:, c:, c]), axis=1)
        ok &= np.abs(A[idx, piv, c]) >= 1e-10
        rc, rp = A[idx, c].copy(), A[idx, piv].copy()
        A[idx, c], A[idx, piv] = rp, rc
        pc = np.where(ok, A[:, c, c], 1.0)
        f = A[:, c + 1:, c] / pc[:, None]
        A[:, c + 1:, :] -= f[..., None] * A[:, c:c + 1, :]
    hn = np.ones(A.shape[:1] + (9,))
    for c in range(7, -1, -1):
        s = A[:, c, 8] - (A[:, c, c + 1:8] * hn[:, c + 1:8]).sum(-1)
        hn[:, c] = s / np.where(ok, A[:, c, c], 1.0)
    with np.errstate(all="ignore"):
        h = denormalise("homography", hn.reshape(-1, 3, 3), t0, t1)
        inv_ok = np.isfinite(h).all((-1, -2)) & (np.linalg.det(np.where(np.isfinite(h), h, 0)) != 0)
    return h, ok & inv_ok


def f_rows(u, u2):
    x, y, x2, y2 = u[..., 0], u[..., 1], u2[..., 0], u2[..., 1]
    return np.stack([x2 * x, x2 * y, x2, y2 * x, y2 * y, y2, x, y, np.ones_like(x)], -1)


def h_rows(u, u2):
    x, y, x2, y2 = u[..., 0], u[..., 1], u2[..., 0], u2[..., 1]
    z, o = np.zeros_like(x), np.ones_like(x)
    a = np.stack([-x, -y, -o, z, z, z, x2 * x, x2 * y, x2], -1)
    b = np.stack([z, z, z, -x, -y, -o, y2 * x, y2 * y, y2], -1)
    return np.concatenate([a, b], -2)


def solve_system(model, m, t0, t1, need_rank):
    w, v = np.linalg.eigh(m)
    ok = w[..., 1] > 1e-12 * w[..., -1] if need_rank else np.ones(w.shape[:-1], bool)
    mn = v[..., :, 0].reshape(v.shape[:-2] + (3, 3))
    if model == "fundamental":
        mn = rank2(mn)
    out = denormalise(model, mn, t0, t1)
    return out, ok & np.isfinite(out).all((-1, -2))


def solve_f8(p0, p1):
    t0, ok0 = norm_t(p0)
    t1, ok1 = norm_t(p1)
    a = f_rows(apply(t0, p0), apply(t1, p1))
    f, ok = solve_system("fundamental", np.swapaxes(a, -1, -2) @ a, t0, t1, True)
    return f, ok & ok0 & ok1


def errors(model, m, p0, p1):
    """m [..., 3, 3], p [n, 2] -> squared pixel errors [..., n] (inf / NaN: never an inlier)."""
    x0, y0, x1, y1 = p0[:, 0], p0[:, 1], p1[:, 0], p1[:, 1]
    m = m[..., None, :, :]
    with np.errstate(all="ignore"):
        if model == "homography":
            mi = np.linalg.inv(m)
            pw = m[..., 2, 0] * x0 + m[..., 2, 1] * y0 + m[..., 2, 2]
            px = (m[..., 0, 0] * x0 + m[..., 0, 1] * y0 + m[..., 0, 2]) / pw - x1
            py = (m[..., 1, 0] * x0 + m[..., 1, 1] * y0 + m[..., 1, 2]) / pw - y1
            qw = mi[..., 2, 0] * x1 + mi[..., 2, 1] * y1 + mi[..., 2, 2]
            qx = (mi[..., 0, 0] * x1 + mi[..., 0, 1] * y1 + mi[..., 0, 2]) / qw - x0
            qy = (mi[..., 1, 0] * x1 + mi[..., 1, 1] * y1 + mi[..., 1, 2]) / qw - y0
            return 0.5 * (px * px + py * py + qx * qx + qy * qy)
        f0 = m[..., 0, 0] * x0 + m[..., 0, 1] * y0 + m[..., 0, 2]
        f1 = m[..., 1, 0] * x0 + m[..., 1, 1] * y0 + m[..., 1, 2]
        f2 = m[..., 2, 0] * x0 + m[..., 2, 1] * y0 + m[..., 2, 2]
        g0 = m[..., 0, 0] * x1 + m[..., 1, 0] * y1 + m[..., 2, 0]
        g1 = m[..., 0, 1] * x1 + m[..., 1, 1] * y1 + m[..., 2, 1]
        e = x1 * f0 + y1 * f1 + f2
        return e * e / (f0 * f0 + f1 * f1 + g0 * g0 + g1 * g1)


def output_scale(model, m):
    nrm = np.linalg.norm(m)
    flat = m.reshape(-1)
    d = nrm if flat[np.argmax(np.abs(flat))] >= 0 else -nrm
    if model == "homography" and abs(m[2, 2]) > 1e-12 * nrm:
        d = m[2, 2]
    return m / d


def ransac_ref(p0, p1, model, thr, iterations, seed=0, pair_id=0):
    """One pair's compacted matches [n, 2] -> dict(best, model [3, 3] (NaN when none), mask [n], count, samples)."""
    p0, p1 = np.asarray(p0, np.float64), np.asarray(p1, np.float64)
    n, s, t2 = len(p0), S[model], float(np.float32(thr)) ** 2
    none = {"best": -1, "model": np.full((3, 3), np.nan), "mask": np.zeros(n, bool), "count": 0, "samples": None}
    if n < s:
        return none
    samples = draw_samples(seed, pair_id, n, s, iterations)
    m, ok = (solve_h4 if model == "homography" else solve_f8)(p0[samples], p1[samples])
    e = errors(model, np.where(ok[:, None, None], m, np.eye(3)), p0, p1)   # degenerate: placeholder, not ranked
    inl = e < t2
    cnt = np.where(ok, inl.sum(1), -1)
    cost = np.where(inl, e, 0).sum(1) + (n - inl.sum(1)) * t2
    if not ok.any():
        return dict(none, samples=samples)
    order = np.lexsort((np.arange(iterations), cost, -cnt))
    best = int(order[0])
    mdl = m[best]
    inl = errors(model, mdl, p0, p1) < t2
    if inl.sum() >= s:
        t0, ok0 = norm_t(p0[inl])
        t1, ok1 = norm_t(p1[inl])
        if ok0 and ok1:
            u, u2 = apply(t0, p0[inl]), apply(t1, p1[inl])
            a = h_rows(u, u2) if model == "homography" else f_rows(u, u2)
            r, rok = solve_system(model, a.T @ a, t0, t1, False)
            if rok and (model == "fundamental" or np.linalg.det(r) != 0):
                mdl = r
    mask = errors(model, mdl, p0, p1) < t2
    return {"best": best, "model": output_scale(model, mdl), "mask": mask, "count": int(mask.sum()),
            "samples": samples}


# ---------------------------------------------------------------------------------------------- synthetic scenes
def random_h(rs):
    return np.array([[1 + rs.uniform(-.2, .2), rs.uniform(-.2, .2), rs.uniform(-60, 60)],
                     [rs.uniform(-.2, .2), 1 + rs.uniform(-.2, .2), rs.uniform(-60, 60)],
                     [rs.uniform(-3e-4, 3e-4), rs.uniform(-3e-4, 3e-4), 1.0]])


def project_h(h, p):
    q = p @ h[:, :2].T + h[:, 2]
    return q[:, :2] / q[:, 2:]


def rot(rs, deg):
    ax = rs.standard_normal(3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(deg)
    k = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(a) * k + (1 - np.cos(a)) * k @ k


def scene(rs, model, n, outlier_ratio, sigma=0.5, w=640, h=480):
    """-> p0, p1 [n, 2] float32, is_inlier [n], ground-truth model, noise-free (p0, p1) of the inliers."""
    n_out = int(round(outlier_ratio * n))
    if model == "homography":
        gt = random_h(rs)
        p0 = rs.uniform((0, 0), (w, h), (n, 2))
        clean1 = project_h(gt, p0)
    else:
        kk = np.array([[500.0, 0, w / 2], [0, 500.0, h / 2], [0, 0, 1]])
        r, t = rot(rs, 8.0), np.array([1.0, rs.uniform(-.3, .3), rs.uniform(-.3, .3)])
        X = np.stack([rs.uniform(-4, 4, n), rs.uniform(-3, 3, n), rs.uniform(6, 14, n)], 1)
        x0 = X @ kk.T
        p0 = x0[:, :2] / x0[:, 2:]
        x1 = (X @ r.T + t) @ kk.T
        clean1 = x1[:, :2] / x1[:, 2:]
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        ki = np.linalg.inv(kk)
        gt = ki.T @ tx @ r @ ki
    clean0 = p0.copy()
    p1 = clean1 + sigma * rs.standard_normal((n, 2))
    p0 = p0 + sigma * rs.standard_normal((n, 2))
    inl = np.ones(n, bool)
    out = rs.permutation(n)[:n_out]
    inl[out] = False
    p1[out] = rs.uniform((0, 0), (w, h), (n_out, 2))
    return p0.astype(np.float32), p1.astype(np.float32), inl, gt, (clean0[inl], clean1[inl])


def pad_batch(pairs, K, rs=None):
    """[(p0, p1)] -> padded [B, K, 2] arrays and a bool mask; with rs the valid entries go to random columns."""
    B = len(pairs)
    P0, P1 = np.full((B, K, 2), 7.0, np.float32), np.full((B, K, 2), -3.0, np.float32)   # junk in the padding
    V = np.zeros((B, K), bool)
    cols = []
    for b, (a, c) in enumerate(pairs):
        col = np.sort(rs.permutation(K)[:len(a)]) if rs is not None else np.arange(len(a))
        P0[b, col], P1[b, col], V[b, col] = a, c, True
        cols.append(col)
    return P0, P1, V, cols


def model_dist(a, b):
    """Distance of two 3x3 models up to scale and sign."""
    a, b = a / np.linalg.norm(a), b / np.linalg.norm(b)
    return min(np.abs(a - b).max(), np.abs(a + b).max())


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
