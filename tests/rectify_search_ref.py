"""Host reference of the rectification search's selection rule (DESIGN.md §20), from per-candidate flags and match
lists.  Candidate c = b * K + k of pair b.  A candidate's count is the number of its rows that pass the flag test
(before any per-pair cap); pair b keeps the smallest k with the largest count (0 when every count is 0), and the
search's match list is the list of the N * K candidate pairs restricted to the chosen candidates, with pair ids b
instead of c."""
import numpy as np
import torch

from match_cap_ref import LIST_KEYS


def counts_from_flags(flags, k):
    """flags [N * K, L] bool (the flag test of every candidate row) -> counts [N, K] int64."""
    f = np.asarray(flags, dtype=bool)
    return f.sum(1).reshape(-1, k)


def counts_from_ids(b_ids, n, k):
    """Candidate ids of an uncapped match list of the N * K candidate pairs (one entry per flagged row) -> counts
    [N, K] int64."""
    b = np.asarray(b_ids.cpu() if torch.is_tensor(b_ids) else b_ids, dtype=np.int64)
    return np.bincount(b, minlength=n * k).reshape(n, k)


def choose(counts):
    """counts [N, K] -> choice [N] int64: per pair, the smallest k with the largest count."""
    counts = np.asarray(counts)
    choice = np.zeros(counts.shape[0], np.int64)
    for b, row in enumerate(counts):
        best = -1
        for k, c in enumerate(row):
            if c > best:   # strictly larger: a tie keeps the earlier k
                best, choice[b] = c, k
    return choice


def winners(lists, choice, k, keys=LIST_KEYS):
    """The entries of a match list of the N * K candidate pairs (dict of tensors with candidate ids in b_ids / m_bids)
    whose candidate is its pair's choice, in list order, with b_ids / m_bids divided by K."""
    choice = torch.as_tensor(np.asarray(choice)).to(lists["b_ids"].device)
    b = lists["b_ids"]
    keep = (b % k) == choice[b // k]
    out = {key: lists[key][keep] for key in keys}
    for key in ("b_ids", "m_bids"):
        if key in out:
            out[key] = out[key] // k
    return out
