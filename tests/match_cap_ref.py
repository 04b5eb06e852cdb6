"""Torch statement of the per-pair match cap (`match_coarse.max_matches_per_pair`), applied to an uncapped output.

Within each pair, the k rows with the largest mconf are kept; a tie at the k-th value goes to the smaller row index i.
The kept rows stay in ascending (b, i) order.  Every list key of a capped forward must equal the same rows of the
uncapped one."""
import torch

# keys of `forward` whose first dimension is the match count
LIST_KEYS = ["b_ids", "i_ids", "j_ids", "m_bids", "gt_mask", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f",
             "expec_f"]


def capped_rows(b_ids, mconf, k):
    """Indices (ascending) of the rows of a (b, i)-ordered list that a cap of k matches per pair keeps."""
    m = b_ids.shape[0]
    if m == 0:
        return torch.zeros(0, dtype=torch.long, device=b_ids.device)
    order = torch.sort(-mconf, stable=True).indices              # by -mconf; ties keep the list's (b, i) order
    order = order[torch.sort(b_ids[order], stable=True).indices]  # grouped by pair, (-mconf, i) order inside
    _, counts = torch.unique_consecutive(b_ids[order], return_counts=True)
    starts = torch.cumsum(counts, 0) - counts
    rank = torch.arange(m, device=b_ids.device) - torch.repeat_interleave(starts, counts)
    return torch.sort(order[rank < k]).values


def apply_cap(out, k):
    """-> the list keys of `out` (an uncapped forward's outputs) restricted to the rows a cap of k keeps.  With
    thr < 0 the mconf != 0 filter has to have removed nothing (the fine stage needs one keypoint per window)."""
    m = out["b_ids"].shape[0]
    assert all(out[key].shape[0] == m for key in LIST_KEYS), "a filtered list key: the selection needs every mconf"
    idx = capped_rows(out["b_ids"], out["mconf"], k)
    return {key: out[key][idx] for key in LIST_KEYS}


def per_pair_counts(b_ids, n):
    return torch.bincount(b_ids, minlength=n).tolist()
