"""Reference statement of `LoFTR.match_points` (DESIGN.md §17): rules 1, 2 and 4 in numpy, and the fine stage of one
set of queries in float64 (or float32, the emulation the project rule compares against) from centre-based windows,
otherwise through tests/ref64.py.  Image1 queries (DESIGN.md §22) use the same rules with the images' roles swapped:
rules 1, 2 and 4 are `query_cells` and `image1_centres` given image1's sizes, scale and mask, rule 3 is
`column_answer`, and the fine stage is `fine_stage(..., side=1)`."""
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


def column_answer(conf, b, j):
    """Rule 3 of image1 queries on a float64 confidence matrix conf [N, L, S]: i = the column arg-max of (b, j) (the
    smallest i of a tie), its conf, and whether (i, j) is mutual (j is the row arg-max of i) -> (i, conf, mutual)."""
    col = conf[b, :, j]   # [M, L]
    i = col.argmax(1)
    c = col.gather(1, i[:, None])[:, 0]
    mutual = conf[b, i].argmax(1) == torch.as_tensor(j, device=conf.device)
    return i, c, mutual


def fine_stage(model, feat_f0, feat_f1, x0, x1, b_ids, i_ids, j_ids, f0, f1, pts_c, hw0_i, scale=None,
               dtype=torch.float64, side=0):
    """FinePreprocess + fine transformer + FineMatching (ref64) of the query windows centred on f0 / f1 [M, 2]:
    feat_f [N, C, h, w], x0 / x1 the coarse transformer outputs [N, L / S, C] (dtype).  The windows pass the merge and
    the fine transformer in (window0, window1) order on either side.  side 0: window0's centre correlated against
    window1, refined from pts_c [M, 2], the image1 window centres in source pixels, with `scale` = scale1.  side 1 (the
    mirrored fine match of image1 queries): window1's centre against window0, refined from the image0 window centres
    with `scale` = scale0 -> (expec_f [M, 3], refined points [M, 2])."""
    dev = feat_f0.device
    cfg = model.config
    W = cfg["fine_window_size"]
    b = torch.as_tensor(b_ids, device=dev)
    i, j = torch.as_tensor(i_ids, device=dev), torch.as_tensor(j_ids, device=dev)
    fw = {k: v.detach().to(dev, dtype) for k, v in model.fine_preprocess.state_dict().items()}
    win0 = centred_windows(feat_f0, b, torch.as_tensor(f0), W)
    win1 = centred_windows(feat_f1, b, torch.as_tensor(f1), W)
    m0, m1 = R.fine_merge(win0, win1, x0[b, i], x1[b, j], W, fw)
    fc = cfg["fine"]
    g0, g1 = R.transformer(m0, m1, R.layer_weights(model.loftr_fine, dev, dtype=dtype),
                           fc["layer_names"], fc["nhead"], attention=fc.get("attention", "linear"))
    if side == 1:
        g0, g1 = g1, g0
    return R.fine_matching(g0, g1, torch.as_tensor(pts_c, device=dev, dtype=dtype), b, hw0_i, feat_f0.shape[2:],
                           scale, dtype)
