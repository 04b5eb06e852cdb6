"""Float64 reference of guided coarse matching (DESIGN.md §18) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The guided confidence matrix is tests/ref64.py's, given `admissible` as its `adm`: inadmissible similarity entries are
filled with -INF (the reference's padding fill, coarse_matching.py:111-123) and their conf is set to 0 before the
selection, which is ref64.coarse_match unchanged.  This module adds what the guide itself needs:
- `coarse_points`: the coarse keypoints mkpts0_c / mkpts1_c of every cell, in float32 as the kernels compute them;
- `admissible`: the guide's predicate, evaluated in float32 with the operation order the kernels use (numpy rounds
  every float32 operation separately, as the kernels' explicitly rounded intrinsics do), so it is bit for bit the
  kernels' predicate; and its float64 distance from the band's edge, to leave near-boundary cell pairs out of a
  comparison."""
from __future__ import annotations

import numpy as np

F32 = np.float32


def coarse_points(n, hw_c, img_scale, scale=None):
    """float32 [n, h*w, 2]: (cell % w, cell // w) * img_scale (* scale[b]), as match_scatter_kernel writes
    mkpts0_c / mkpts1_c.  scale: optional [n, 2]."""
    h, w = hw_c
    cells = np.arange(h * w)
    xy = np.stack([cells % w, cells // w], -1).astype(F32)                         # [h*w, 2]
    s = np.full((n, 2), img_scale, F32)
    if scale is not None:
        s = F32(img_scale) * np.asarray(scale, F32)
    return xy[None] * s[:, None, :]


def admissible(kind, model, radius, p0, p1):
    """-> (adm bool [n, L, S], margin float64 [n, L, S]).  kind: "fundamental" | "homography"; model [n, 3, 3];
    p0 [n, L, 2], p1 [n, S, 2] float32 (coarse_points).  margin: |distance - radius| in float64 (the point-line
    distance for F, the transfer distance for H); inf for pairs that are unguided or admit nothing."""
    T = np.asarray(model, F32)
    r = F32(radius)
    finite = np.isfinite(T).all(axis=(1, 2))
    x0, y0 = p0[..., 0], p0[..., 1]                                                 # [n, L]
    x1, y1 = p1[:, None, :, 0], p1[:, None, :, 1]                                  # [n, 1, S]
    with np.errstate(all="ignore"):
        v = [((T[:, k, 0, None] * x0 + T[:, k, 1, None] * y0) + T[:, k, 2, None])[:, :, None] for k in range(3)]
        if kind == "fundamental":
            a, b, c = v
            e = (a * x1 + b * y1) + c
            adm = (np.abs(e) <= r * np.sqrt(a * a + b * b)) & ~((a == 0) & (b == 0))
            a64, b64 = a.astype(np.float64), b.astype(np.float64)
            dist = np.abs(e.astype(np.float64)) / np.sqrt(a64 * a64 + b64 * b64)
        elif kind == "homography":
            q2 = v[2]
            dx, dy = v[0] / q2 - x1, v[1] / q2 - y1
            adm = ((dx * dx + dy * dy) <= r * r) & (q2 != 0)
            dist = np.sqrt(dx.astype(np.float64) ** 2 + dy.astype(np.float64) ** 2)
        else:
            raise ValueError(kind)
        margin = np.abs(dist - float(radius))
    margin = np.where(np.isfinite(margin), margin, np.inf)
    adm = np.where(finite[:, None, None], adm, True)
    margin = np.where(finite[:, None, None], margin, np.inf)
    return adm, margin

