"""float64 reference and error rule of the epipolar-error kernel (epipolar_error_kernel, `loftr_b200.evaluation.
compute_symmetrical_epipolar_errors`), plus the synthetic scenes of tests/test_evaluation_edges_gpu.py.

The reference is oracle/metrics_oracle.symmetrical_epipolar_errors: run on float64 copies of the float32 inputs it is
the float64 result r, run on the float32 inputs themselves it is the fp32 oracle.  Each match is judged by its own
conditioning:

    e = |k - r| / (2 |pep| P w + r)

with, from the float64 run, pep = p1^T E p0, w = 1 / |(E p0)_xy|^2 + 1 / |(E^T p1)_xy|^2 and P = |p1|^T |[t]_x| |R| |p0|
(the forward-error scale of the bilinear form, the construction of E = [t]_x R included).  A result within a few
roundings of the float64 one has e of a few 2^-24; the kernel must stay within 4x of the fp32 oracle's largest e."""
import numpy as np

from oracle import metrics_oracle as MO

ULP = 2.0 ** -24


def skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def terms(sc):
    """-> r (float64 errors, NaN for a match outside [0, n_pairs) as the kernel documents) and the per-match scale
    2 |pep| P w + r of the rule."""
    f = {k: np.asarray(v, np.float64) for k, v in sc.items() if k != "m_bids"}
    bids = np.asarray(sc["m_bids"])
    n = len(bids)
    r, scale = np.full(n, np.nan), np.full(n, np.nan)
    for b in range(f["T_0to1"].shape[0]):
        sel = bids == b
        if not sel.any():
            continue
        T, K0, K1 = f["T_0to1"][b], f["K0"][b], f["K1"][b]
        p0 = np.concatenate([(f["mkpts0_f"][sel] - K0[[0, 1], [2, 2]]) / K0[[0, 1], [0, 1]], np.ones((sel.sum(), 1))], 1)
        p1 = np.concatenate([(f["mkpts1_f"][sel] - K1[[0, 1], [2, 2]]) / K1[[0, 1], [0, 1]], np.ones((sel.sum(), 1))], 1)
        E = MO.essential_from_pose(T)
        ep0, etp1 = p0 @ E.T, p1 @ E
        with np.errstate(all="ignore"):
            pep = (p1 * ep0).sum(1)
            w = 1 / (ep0[:, 0] ** 2 + ep0[:, 1] ** 2) + 1 / (etp1[:, 0] ** 2 + etp1[:, 1] ** 2)
            P = ((np.abs(p1) @ (np.abs(skew(T[:3, 3])) @ np.abs(T[:3, :3]))) * np.abs(p0)).sum(1)
            r[sel] = pep ** 2 * w
            scale[sel] = 2 * np.abs(pep) * P * w + r[sel]
    return r, scale


def rule_error(k, r, scale):
    """e per match (NaN where r is NaN)."""
    with np.errstate(all="ignore"):
        return np.abs(np.asarray(k, np.float64) - r) / scale


def oracle32(sc):
    """The fp32 oracle: the float64 reference's arithmetic on the float32 inputs."""
    return MO.symmetrical_epipolar_errors(*(np.asarray(sc[k]) for k in ("mkpts0_f", "mkpts1_f", "m_bids", "T_0to1",
                                                                       "K0", "K1")))


# ------------------------------------------------------------------------------------------------ scenes
def _rot(rs, scale):
    w = rs.standard_normal(3) * scale
    th = np.linalg.norm(w)
    k = skew(w / max(th, 1e-12))
    return np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * k @ k


def _batch(pairs):
    """[(p0 [n, 2], p1 [n, 2], T [4, 4], K0, K1)] -> the float32 batch dict of compute_symmetrical_epipolar_errors."""
    f = np.float32
    return {"mkpts0_f": np.concatenate([p[0] for p in pairs]).astype(f),
            "mkpts1_f": np.concatenate([p[1] for p in pairs]).astype(f),
            "m_bids": np.concatenate([np.full(len(p[0]), b) for b, p in enumerate(pairs)]).astype(np.int64),
            "T_0to1": np.stack([p[2] for p in pairs]).astype(f), "K0": np.stack([p[3] for p in pairs]).astype(f),
            "K1": np.stack([p[4] for p in pairs]).astype(f)}


def _pair(rs, n, R, t, K0, K1, depth, w, h, noise=0.5, outliers=0.1, p0=None):
    """n matches of points in front of both cameras (p0 given: pixels of image 0, else uniform over it)."""
    if p0 is None:
        p0 = rs.uniform((0, 0), (w, h), (n, 2))
    z = rs.uniform(*depth, n)
    X = np.concatenate([(p0 - K0[[0, 1], [2, 2]]) / K0[[0, 1], [0, 1]], np.ones((n, 1))], 1) * z[:, None]
    x1 = (X @ R.T + t) @ K1.T
    p1 = x1[:, :2] / x1[:, 2:] + rs.standard_normal((n, 2)) * noise
    bad = rs.rand(n) < outliers
    p1[bad] = rs.uniform((0, 0), (w, h), (bad.sum(), 2))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return p0, p1, T, K0, K1


def outdoor_scene(seed, n=400):
    """1600x1200 views with |t| from 1e-4 to 1e3 (depths scaled with |t|), one pair per magnitude."""
    rs = np.random.RandomState(seed)
    K = np.array([[1400.0, 0, 800], [0, 1400.0, 600], [0, 0, 1]])
    pairs = []
    for mag in np.logspace(-4, 3, 8):
        t = rs.standard_normal(3)
        t *= mag / np.linalg.norm(t)
        pairs.append(_pair(rs, n, _rot(rs, 0.1), t, K, K * [[1.01], [0.99], [1]], (8 * mag, 60 * mag), 1600, 1200))
    return _batch(pairs)


def forward_scene(seed, n=400):
    """Forward motion: the epipole near the principal point and matches from 0.5 to 40 px around it."""
    rs = np.random.RandomState(seed)
    K = np.array([[600.0, 0, 320], [0, 592.0, 240], [0, 0, 1]])
    pairs = []
    for lateral in (0.0, 0.01, 0.05):
        t = np.array([lateral, -lateral / 2, 1.0])
        e = K @ t
        rad, ang = rs.uniform(0.5, 40, n), rs.uniform(0, 2 * np.pi, n)
        p0 = e[:2] / e[2] + np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)
        pairs.append(_pair(rs, n, _rot(rs, 0.002), t, K, K, (3, 20), 640, 480, p0=p0))
    return _batch(pairs)


def rotation_scene(seed, n=200):
    """Pure rotation (t = 0) next to a translating pair: E = 0 gives NaN in float64, and so must the kernel."""
    rs = np.random.RandomState(seed)
    K = np.array([[580.0, 0, 320], [0, 580.0, 240], [0, 0, 1]])
    pairs = [_pair(rs, n, _rot(rs, 0.2), np.zeros(3), K, K, (2, 8), 640, 480),
             _pair(rs, n, _rot(rs, 0.2), np.array([0.3, 0.1, -0.1]), K, K, (2, 8), 640, 480)]
    return _batch(pairs)


def sized_scene(seed, M):
    """M matches over three ScanNet-like pairs."""
    rs = np.random.RandomState(seed)
    K = np.array([[577.0, 0, 319.5], [0, 571.0, 239.5], [0, 0, 1]])
    sizes = np.diff(np.sort(np.concatenate([[0, M], rs.randint(0, M + 1, 2)])))
    return _batch([_pair(rs, int(m), _rot(rs, 0.25), rs.standard_normal(3) * 0.4, K, K, (2, 8), 640, 480)
                   for m in sizes])
