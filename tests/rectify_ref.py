"""float64 references of rectified matching (DESIGN.md §19): the warp of image1 onto image0's canvas through a per-pair
homography, built on torch.nn.functional.grid_sample (bilinear, zero padding, align_corners=True), and the
back-mapping of rectified points into image1 with its inside flag.  Both apply the kernels' model rules: a model with a
non-finite entry is the identity, and H is multiplied by the sign of w at the centre of image0's canvas."""
import numpy as np
import torch
import torch.nn.functional as F


def _f64(x):
    return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x.detach().cpu()).to(torch.float64)


def _scales(scale, n):
    return torch.ones(n, 2, dtype=torch.float64) if scale is None else _f64(scale).reshape(n, 2)


def effective_models(models, hw0, scale0=None):
    """[N, 3, 3] float64 models as the kernels apply them for image0's canvas hw0 = (H0, W0)."""
    h = _f64(models).reshape(-1, 3, 3).clone()
    n = h.shape[0]
    s0 = _scales(scale0, n)
    bad = ~torch.isfinite(h).flatten(1).all(1)
    h[bad] = torch.eye(3, dtype=torch.float64)
    cx, cy = 0.5 * (hw0[1] - 1) * s0[:, 0], 0.5 * (hw0[0] - 1) * s0[:, 1]
    wc = h[:, 2, 0] * cx + h[:, 2, 1] * cy + h[:, 2, 2]
    h[wc < 0] *= -1
    return h


def warp(image1, models, hw, scale0=None, scale1=None):
    """image1 [N, 1, H1, W1] resampled onto the canvas hw = (H, W) in float64 -> (warp [N, 1, H, W], u, v [N, H, W]:
    the sample positions in image1's pixels, NaN where w <= 0)."""
    img = _f64(image1)
    n, _, h1, w1 = img.shape
    H, W = hw
    hm = effective_models(models, hw, scale0)
    s0, s1 = _scales(scale0, n), _scales(scale1, n)
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    px, py = x[None] * s0[:, 0, None, None], y[None] * s0[:, 1, None, None]
    q = [hm[:, k, 0, None, None] * px + hm[:, k, 1, None, None] * py + hm[:, k, 2, None, None] for k in range(3)]
    ok = q[2] > 0
    u = torch.where(ok, q[0] / q[2] / s1[:, 0, None, None], torch.nan)
    v = torch.where(ok, q[1] / q[2] / s1[:, 1, None, None], torch.nan)
    # far-away and horizon samples become a position well outside the image: grid_sample then reads only padding
    gu = torch.nan_to_num(u, nan=-4.0).clamp(-4.0, w1 + 3.0)
    gv = torch.nan_to_num(v, nan=-4.0).clamp(-4.0, h1 + 3.0)
    grid = torch.stack([2 * gu / (w1 - 1) - 1, 2 * gv / (h1 - 1) - 1], -1)
    out = F.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=True)
    return out, u, v


def near_pixel_boundary(u, v, eps=1e-9):
    """Samples whose position lies within eps of an integer coordinate without being on it: there the floor of the
    kernel's fp64 position may differ from the reference's."""
    def near(t):
        d = (t - torch.round(t)).abs()
        return (d > 0) & (d < eps)
    return near(u) | near(v)


def map_back(pts, ids, models, hw0, hw1, scale0=None, scale1=None, mask1=None):
    """Points [m, 2] of the rectified frame (source pixels of image0's) of pairs ids [m] -> (float64 [m, 2] in source
    pixels of image1, NaN where w <= 0 or the point is not finite; inside [m] bool: in [0, W1 - 1] x [0, H1 - 1] in
    image1's pixels and, with mask1 [N, H1/8, W1/8], in a true cell)."""
    p = _f64(pts).reshape(-1, 2)
    ids = torch.as_tensor(np.asarray(ids) if not torch.is_tensor(ids) else ids.cpu()).long()
    n = _f64(models).reshape(-1, 9).shape[0]
    hm = effective_models(models, hw0, scale0)[ids]
    s1 = _scales(scale1, n)[ids]
    q = [hm[:, k, 0] * p[:, 0] + hm[:, k, 1] * p[:, 1] + hm[:, k, 2] for k in range(3)]
    ok = q[2] > 0
    x = torch.where(ok, q[0] / q[2], torch.nan)
    y = torch.where(ok, q[1] / q[2], torch.nan)
    u, v = x / s1[:, 0], y / s1[:, 1]
    inside = ok & (u >= 0) & (u <= hw1[1] - 1) & (v >= 0) & (v <= hw1[0] - 1)
    if mask1 is not None and inside.any():
        m1 = torch.as_tensor(np.asarray(mask1) if not torch.is_tensor(mask1) else mask1.cpu()).bool()
        k = inside.nonzero()[:, 0]
        inside[k] = m1[ids[k], torch.floor(v[k] / 8).long(), torch.floor(u[k] / 8).long()]
    return torch.stack([x, y], 1), inside
