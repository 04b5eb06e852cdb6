"""float64 NumPy implementation of the robust two-view geometry estimator (`loftr_b200.estimate_geometry`,
csrc/geometry.cuh), shared by tests/test_geometry.py and tests/test_geometry_edges_gpu.py.

The same Philox4x32-10 sample draw, the same minimal solvers (4-point normalised DLT with h33 = 1; normalised 8-point
with rank 2), the same errors (symmetric transfer, Sampson), the same MSAC ranking and the same Hartley-normalised
least-squares refit.  The GPU runs the geometry in fp64 too, so on identical samples the winning hypothesis must agree
exactly and the refitted model to rounding.  `tile_ranking` gives the winner of every 64-hypothesis scoring tile and
`ws_layout` mirrors the workspace the library carves, so a test can read the kernels' intermediate results back.
Also here: the synthetic scenes with known H / F and the padded [B, K] layout."""
import numpy as np

S = {"homography": 4, "fundamental": 8}
HYP_PER_TILE = 64      # kGeoHypPerBlock: hypotheses per scoring block (one tile_best entry each)
STAGE = 1024           # kGeoStage: matches staged in shared memory per round of the scoring loop
GEO_BEST = np.dtype([("sum", "<f8"), ("count", "<i4"), ("hyp", "<i4")])   # struct GeoBest, 16 bytes


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
    """[iterations, s] ascending indices in [0, n): the kernel's draw (header of lb_estimate_geometry).  pair_id is the
    32-bit counter word the kernel uses (estimate_geometry keys a pair with its id modulo 2**32)."""
    assert 0 <= pair_id < 2 ** 32, pair_id
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
    ata = np.swapaxes(a, -1, -2) @ a
    ata = np.where(np.isfinite(ata).all((-1, -2))[..., None, None], ata, np.eye(9))   # non-finite: not ok0 / ok1
    f, ok = solve_system("fundamental", ata, t0, t1, True)
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


def score_hypotheses(p0, p1, model, thr, iterations, seed=0, pair_id=0, upto=None):
    """Every hypothesis of one pair's compacted matches [n, 2] (n >= s) as the scoring kernel ranks it -> dict(samples
    [it, s], model [it, 3, 3], ok [it], count [it] (-1: degenerate), cost [it] (MSAC; 0 when degenerate)).  upto: score
    against the first `upto` matches only (samples still come from all n), a model of a scoring loop that stops early."""
    p0, p1 = np.asarray(p0, np.float64), np.asarray(p1, np.float64)
    n, s, t2 = len(p0), S[model], float(np.float32(thr)) ** 2
    samples = draw_samples(seed, pair_id, n, s, iterations)
    with np.errstate(all="ignore"):
        m, ok = (solve_h4 if model == "homography" else solve_f8)(p0[samples], p1[samples])
    e = errors(model, np.where(ok[:, None, None], m, np.eye(3)), p0[:upto], p1[:upto])   # degenerate: placeholder
    inl = e < t2
    cnt = np.where(ok, inl.sum(1), -1)
    cost = np.where(ok, np.where(inl, e, 0).sum(1) + (n - inl.sum(1)) * t2, 0.0)
    return {"samples": samples, "model": m, "ok": ok, "count": cnt, "cost": cost,
            "cost_rtol": cost_rtol(model, p0[samples], p1[samples])}


def cost_rtol(model, p0, p1):
    """Relative tolerance of a hypothesis' MSAC cost between two fp64 implementations, per sample [..., s, 2].  The
    kernel sums each staging round in order and NumPy pairwise: 1e-12.  The 8-point null vector comes from another
    eigensolver (cyclic Jacobi against LAPACK) and is only determined to about eps * lambda_max / lambda_2 of the
    normalised A^T A; 32x that covers the cost movement measured between two LAPACK solvers (at most 8.6x)."""
    base = np.full(p0.shape[:-2], 1e-12)
    if model == "homography":
        return base
    with np.errstate(all="ignore"):
        t0, _ = norm_t(p0)
        t1, _ = norm_t(p1)
        a = f_rows(apply(t0, p0), apply(t1, p1))
        ata = np.swapaxes(a, -1, -2) @ a
        ata = np.where(np.isfinite(ata).all((-1, -2))[..., None, None], ata, np.eye(9))
        w = np.linalg.eigvalsh(ata)
        kappa = np.where(w[..., 1] > 0, w[..., -1] / w[..., 1], np.inf)
    return np.maximum(base, 32 * np.finfo(np.float64).eps * kappa)


def ransac_ref(p0, p1, model, thr, iterations, seed=0, pair_id=0):
    """One pair's compacted matches [n, 2] -> dict(best, model [3, 3] (NaN when none), mask [n], count, samples)."""
    p0, p1 = np.asarray(p0, np.float64), np.asarray(p1, np.float64)
    n, s, t2 = len(p0), S[model], float(np.float32(thr)) ** 2
    none = {"best": -1, "model": np.full((3, 3), np.nan), "mask": np.zeros(n, bool), "count": 0, "samples": None}
    if n < s:
        return none
    h = score_hypotheses(p0, p1, model, thr, iterations, seed, pair_id)
    samples, m, ok, cnt, cost = h["samples"], h["model"], h["ok"], h["count"], h["cost"]
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


def staged_scene(rs, model, n, sigma=0.5):
    """-> p0, p1 [n, 2] float32 compacted matches whose scoring rounds (STAGE matches each) disagree.  For n >= 2 STAGE
    the first round holds a weak structure (40 % inliers of one model among outliers) and every later match is an
    inlier of another, dominant model, so ranking only the first round picks another winner.  Below that, one
    structure with 30 % outliers; the match at index STAGE (the lone match of the second round at n = STAGE + 1) is
    one of its inliers."""
    if n >= 2 * STAGE:
        a0, a1 = scene(rs, model, STAGE, 0.6, sigma)[:2]
        b0, b1 = scene(rs, model, n - STAGE, 0.0, sigma)[:2]
        return np.concatenate([a0, b0]), np.concatenate([a1, b1])
    p0, p1, inl = scene(rs, model, n, 0.3, sigma)[:3]
    if n > STAGE and not inl[STAGE]:
        j = np.flatnonzero(inl)[0]
        for p in (p0, p1):
            p[[j, STAGE]] = p[[STAGE, j]]
    return p0, p1


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


def tile_ranking(p0, p1, model, thr, iterations, seed=0, pair_id=0, upto=None):
    """The winner of every 64-hypothesis tile under geo_better (more inliers, then lower cost, then lower index), as
    geometry_score_kernel stores it in tile_best -> (count, cost, hyp) arrays [n_tiles], plus the scores of every
    hypothesis.  A tile whose hypotheses are all degenerate (or a pair below the sample size) holds count -1, cost 0
    and the tile's first index."""
    n, s = len(p0), S[model]
    n_tiles = -(-iterations // HYP_PER_TILE)
    pad = n_tiles * HYP_PER_TILE
    cnt, cost = np.full(pad, -1, np.int64), np.zeros(pad)
    h = None
    if n >= s:
        h = score_hypotheses(p0, p1, model, thr, iterations, seed, pair_id, upto)
        cnt[:iterations], cost[:iterations] = h["count"], h["cost"]
    hyp = np.arange(pad)
    order = np.lexsort((hyp.reshape(n_tiles, -1), cost.reshape(n_tiles, -1), -cnt.reshape(n_tiles, -1)), axis=1)
    win = order[:, 0] + np.arange(n_tiles) * HYP_PER_TILE
    return cnt[win], cost[win], win, h


def ws_layout(B, K, iterations):
    """Byte offsets of the workspace lb_estimate_geometry carves (geometry_ws_layout in engine.cu): compact [B, K]
    float4, compact_col [B, K] int32, n_valid [B] int32 and tile_best [B, n_tiles] GeoBest, each region 16-byte
    aligned -> dict of offsets and "total" (what lb_geometry_workspace_bytes returns; 0 for an empty call)."""
    if B <= 0 or K <= 0 or iterations <= 0:
        return {"total": 0}
    up16 = lambda x: (x + 15) & ~15
    n_tiles = -(-iterations // HYP_PER_TILE)
    compact_col = B * K * 16
    n_valid = compact_col + up16(B * K * 4)
    tile_best = n_valid + up16(B * 4)
    return {"compact": 0, "compact_col": compact_col, "n_valid": n_valid, "tile_best": tile_best, "n_tiles": n_tiles,
            "total": tile_best + B * n_tiles * GEO_BEST.itemsize}


# the staging grid of tests/test_geometry_edges_gpu.py: per-pair match counts n (the last one is the matcher's largest
# per-pair count, 1280x960 at 1/8: L = 19200), each pair alone in a row of K = max(n, 19200 if n == 19200 else n + 61)
STAGING_N = (1023, 1024, 1025, 2048, 2049, 4100, 19200)
STAGING_THR = 3.0


def staging_case(model, n):
    """-> p0, p1 (compacted, float32), iterations, seed of the staging grid point (model, n)."""
    rs = np.random.RandomState(n + 7 * S[model])
    p0, p1 = staged_scene(rs, model, n)
    iterations = 256 if n == 19200 else 320 if model == "homography" else 1024
    return p0, p1, iterations, 1000 + n
