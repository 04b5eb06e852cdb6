"""Reference statement of image1-side point queries (DESIGN.md §22): rules 1-5 with the roles of the images swapped, in
numpy / float64, on top of tests/points_ref.py.  Rules 1, 2 and 4 are points_ref's with image1's sizes and mask; rule 3
reads a float64 confidence matrix by column; rule 5 correlates window1's centre against window0."""
import torch

import points_ref as P
import ref64 as R

query_cells = P.query_cells   # rules 1 and 2 on image1: pass hw1_* sizes, scale1 and mask1


def image0_centres(cell1, f1, i, w0c, stride):
    """Rule 4 on image0: f0 = stride * (ix, iy) + f1 - stride * (jx, jy)."""
    return P.image1_centres(cell1, f1, i, w0c, stride)


def column_answer(conf, b, j):
    """Rule 3 on a float64 confidence matrix conf [N, L, S]: i = the column arg-max of (b, j) (the smallest i of a
    tie), its conf, and whether (i, j) is mutual (j is the row arg-max of i) -> (i, conf, mutual) arrays."""
    col = conf[b, :, j]   # [M, L]
    i = col.argmax(1)
    c = col.gather(1, i[:, None])[:, 0]
    mutual = conf[b, i].argmax(1) == torch.as_tensor(j, device=conf.device)
    return i, c, mutual


def fine_stage_back(model, feat_f0, feat_f1, x0, x1, b_ids, i_ids, j_ids, f0, f1, pts0_c, hw0_i, scale0=None,
                    dtype=torch.float64):
    """The fine stage of image1 queries: windows centred on f0 / f1 [M, 2] through FinePreprocess and the fine
    transformer in (window0, window1) order, exactly as points_ref.fine_stage, then the mirrored fine match: window1's
    centre correlated against window0, the expectation over window0, refined from pts0_c [M, 2] with scale0
    -> (expec_f [M, 3], pts0_f [M, 2])."""
    dev = feat_f0.device
    cfg = model.config
    W = cfg["fine_window_size"]
    b = torch.as_tensor(b_ids, device=dev)
    i, j = torch.as_tensor(i_ids, device=dev), torch.as_tensor(j_ids, device=dev)
    fw = {k: v.detach().to(dev, dtype) for k, v in model.fine_preprocess.state_dict().items()}
    win0 = P.centred_windows(feat_f0, b, torch.as_tensor(f0), W)
    win1 = P.centred_windows(feat_f1, b, torch.as_tensor(f1), W)
    c_win = torch.cat([x0[b, i], x1[b, j]], 0) @ fw["down_proj.weight"].T + fw["down_proj.bias"]
    cat = torch.cat([torch.cat([win0, win1], 0), c_win[:, None].expand(-1, W * W, -1)], -1)
    merged = cat @ fw["merge_feat.weight"].T + fw["merge_feat.bias"]
    m = len(b)
    fc = cfg["fine"]
    g0, g1 = R.transformer(merged[:m], merged[m:], R.layer_weights(model.loftr_fine, dev, dtype=dtype),
                           fc["layer_names"], fc["nhead"], attention=fc.get("attention", "linear"))
    return P._fine_matching(g1, g0, torch.as_tensor(pts0_c, device=dev, dtype=dtype), b, hw0_i, feat_f0.shape[2:],
                            scale0, dtype)
