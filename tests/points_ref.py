"""Reference statement of `LoFTR.match_points` (DESIGN.md §17): rules 1, 2 and 4 in numpy, and the fine stage of one
set of queries in float64 (or float32, the emulation the project rule compares against) from centre-based windows,
otherwise through tests/ref64.py."""
import math

import numpy as np
import torch

import ref64 as R


def query_cells(points, valid, hw_i, hw_c, hw_f, scale0=None, mask0=None):
    """Rules 1 (without the row test of rule 3), 2 and 4 for one pair: points [Q, 2] (source pixels when scale0 [2] is
    given), valid [Q] bool or None, mask0 [h_c, w_c] bool or None.
    -> inside [Q] bool, cell (cx, cy) [Q, 2] int, fine centre f0 [Q, 2] int (both 0 where not inside)."""
    (H0, W0), (h_c, w_c), (h_f, w_f) = hw_i, hw_c, hw_f
    s_c, s_f = H0 / h_c, H0 / h_f
    p = np.asarray(points, np.float32)
    if scale0 is not None:
        p = p / np.asarray(scale0, np.float32)
    with np.errstate(invalid="ignore"):
        inside = np.isfinite(p).all(1) & (p[:, 0] >= 0) & (p[:, 0] <= W0 - 1) & (p[:, 1] >= 0) & (p[:, 1] <= H0 - 1)
    if valid is not None:
        inside &= np.asarray(valid, bool)
    q = np.where(inside[:, None], p, 0).astype(np.float32)
    cell = np.stack([np.clip(np.floor(q[:, 0] / np.float32(s_c) + np.float32(0.5)), 0, w_c - 1),
                     np.clip(np.floor(q[:, 1] / np.float32(s_c) + np.float32(0.5)), 0, h_c - 1)], 1).astype(np.int64)
    if mask0 is not None:
        inside &= np.asarray(mask0, bool)[cell[:, 1], cell[:, 0]]
    f0 = np.stack([np.clip(np.floor(q[:, 0] / np.float32(s_f) + np.float32(0.5)), 0, w_f - 1),
                   np.clip(np.floor(q[:, 1] / np.float32(s_f) + np.float32(0.5)), 0, h_f - 1)], 1).astype(np.int64)
    cell[~inside] = 0
    f0[~inside] = 0
    return inside, cell, f0


def image1_centres(cell, f0, j, w1c, stride):
    """Rule 4 on image1: f1 = stride * (jx, jy) + f0 - stride * (cx, cy)."""
    j = np.asarray(j, np.int64)
    jc = np.stack([j % w1c, j // w1c], 1)
    return stride * jc + np.asarray(f0) - stride * np.asarray(cell)


def centred_windows(feat_f, b_ids, centres, W):
    """Windows W x W centred on fine pixels (x, y) of feat_f [N, C, H, W], zero outside -> [M, WW, C]: the reference's
    unfold padding, with the window placed at any fine pixel instead of at stride * cell."""
    n, c, h, w = feat_f.shape
    r = W // 2
    pad = torch.nn.functional.pad(feat_f, (r, r, r, r))
    out = []
    for b, (x, y) in zip(b_ids.tolist(), centres.tolist()):
        win = torch.zeros(c, W, W, dtype=feat_f.dtype, device=feat_f.device)
        y0, x0 = y, x   # padded coordinates of the window's first row / column
        ys, xs = slice(max(y0, 0), min(y0 + W, h + 2 * r)), slice(max(x0, 0), min(x0 + W, w + 2 * r))
        win[:, ys.start - y0:ys.stop - y0, xs.start - x0:xs.stop - x0] = pad[b, :, ys, xs]
        out.append(win.reshape(c, W * W).T)
    return torch.stack(out) if out else feat_f.new_zeros(0, W * W, c)


def fine_stage(model, feat_f0, feat_f1, x0, x1, b_ids, i_ids, j_ids, f0, f1, pts1_c, hw0_i, scale1=None,
               dtype=torch.float64):
    """FinePreprocess + fine transformer + FineMatching (ref64) of the query windows centred on f0 / f1 [M, 2]:
    feat_f [N, C, h, w], x0 / x1 the coarse transformer outputs [N, L / S, C] (dtype), pts1_c [M, 2] the image1
    window centres in source pixels -> (expec_f [M, 3], pts1_f [M, 2])."""
    dev = feat_f0.device
    cfg = model.config
    W = cfg["fine_window_size"]
    b = torch.as_tensor(b_ids, device=dev)
    i, j = torch.as_tensor(i_ids, device=dev), torch.as_tensor(j_ids, device=dev)
    fw = {k: v.detach().to(dev, dtype) for k, v in model.fine_preprocess.state_dict().items()}
    win0 = centred_windows(feat_f0, b, torch.as_tensor(f0), W)
    win1 = centred_windows(feat_f1, b, torch.as_tensor(f1), W)
    c_win = torch.cat([x0[b, i], x1[b, j]], 0) @ fw["down_proj.weight"].T + fw["down_proj.bias"]
    cat = torch.cat([torch.cat([win0, win1], 0), c_win[:, None].expand(-1, W * W, -1)], -1)
    merged = cat @ fw["merge_feat.weight"].T + fw["merge_feat.bias"]
    m = len(b)
    fc = cfg["fine"]
    g0, g1 = R.transformer(merged[:m], merged[m:], R.layer_weights(model.loftr_fine, dev, dtype=dtype),
                           fc["layer_names"], fc["nhead"], attention=fc.get("attention", "linear"))
    return _fine_matching(g0, g1, torch.as_tensor(pts1_c, device=dev, dtype=dtype), b, hw0_i, feat_f0.shape[2:],
                          scale1, dtype)


def _fine_matching(f0, f1, mkpts1_c, b_ids, hw0_i, hw0_f, scale1, dtype):
    """ref64.fine_matching in `dtype` (ref64's version is float64 only)."""
    if dtype == torch.float64:
        return R.fine_matching(f0, f1, mkpts1_c, b_ids, hw0_i, hw0_f, scale1)
    m, ww, c = f0.shape
    W = int(math.isqrt(ww))
    sim = torch.einsum("mc,mrc->mr", f0[:, ww // 2], f1)
    heat = torch.softmax(sim / c ** 0.5, dim=1)
    lin = torch.linspace(-1, 1, W, dtype=dtype, device=f0.device)
    grid = torch.stack([lin[None, :].expand(W, W), lin[:, None].expand(W, W)], -1).reshape(ww, 2)
    coords = heat @ grid
    std = torch.sqrt(torch.clamp(heat @ grid ** 2 - coords ** 2, min=1e-10)).sum(-1)
    scale = hw0_i[0] / hw0_f[0]
    s1 = scale * torch.as_tensor(scale1, device=f0.device, dtype=dtype)[b_ids] if scale1 is not None else scale
    return torch.cat([coords, std[:, None]], -1), mkpts1_c + coords * (W // 2) * s1
