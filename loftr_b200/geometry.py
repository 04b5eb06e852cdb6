"""Robust two-view geometry on the GPU: one homography or fundamental matrix per matched pair, with its inlier mask.

`estimate_geometry` fits every pair of a batch in three kernel launches (lb_estimate_geometry): a fixed budget of
RANSAC hypotheses per pair drawn from a counter-based RNG, MSAC scoring against all of the pair's matches, and one
Hartley-normalised least-squares refit on the best hypothesis' inliers.  It takes the padded [B, K] layout (K matches
per pair, a valid mask or count marking the real ones) and does not synchronise with the host, so it can run inside a
captured CUDA graph.  `LoFTR.match_features(..., estimate=...)` runs it on the matcher's own output.
"""
from __future__ import annotations

import ctypes as C
import numbers

import torch

from . import _lib

MODELS = {"homography": _lib.GEOMETRY_HOMOGRAPHY, "fundamental": _lib.GEOMETRY_FUNDAMENTAL}
SAMPLE_SIZE = {"homography": 4, "fundamental": 8}
DEFAULT_ITERATIONS = 2048
DEFAULT_THRESHOLD = 3.0


def _stream(t):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def check_options(model="homography", threshold=DEFAULT_THRESHOLD, iterations=DEFAULT_ITERATIONS, seed=0):
    """Validated (model name, threshold, iterations, seed) of `estimate_geometry`; raises ValueError / TypeError."""
    if model not in MODELS:
        raise ValueError(f"estimate_geometry: model must be one of {sorted(MODELS)} (got {model!r})")
    if isinstance(threshold, bool) or not isinstance(threshold, numbers.Real) or not threshold > 0 \
            or threshold == float("inf"):
        raise ValueError(f"estimate_geometry: threshold must be a positive number of pixels (got {threshold!r})")
    if isinstance(iterations, bool) or not isinstance(iterations, numbers.Integral) or not 1 <= iterations < 2 ** 31:
        raise ValueError(f"estimate_geometry: iterations must be an int in [1, 2**31) (got {iterations!r})")
    if isinstance(seed, bool) or not isinstance(seed, numbers.Integral) or not 0 <= seed < 2 ** 64:
        raise ValueError(f"estimate_geometry: seed must be an int in [0, 2**64) (got {seed!r})")
    return model, float(threshold), int(iterations), int(seed)


@torch.no_grad()
def estimate_geometry(points0, points1, valid=None, model="homography", threshold=DEFAULT_THRESHOLD,
                      iterations=DEFAULT_ITERATIONS, seed=0, pair_ids=None, return_details=False):
    """Fits x1 ~ H x0 (model="homography") or x1^T F x0 = 0 (model="fundamental") to each pair's matches.

    points0, points1: float32 CUDA tensors [B, K, 2] of (x, y) pixel coordinates, pair b's candidate matches being
    (points0[b, k], points1[b, k]).  valid: None (all K are matches), a bool [B, K] mask, or an integer [B] count (the
    first count[b] entries of row b are matches).  K must be at least the minimal sample (4 for H, 8 for F).
    threshold: inlier threshold in pixels, on the symmetric transfer error for H (the root of the mean of the squared
    forward and backward transfer distances) and on the Sampson distance for F.  iterations: hypotheses per pair (a
    fixed budget: there is no adaptive early stop).  seed and pair_ids (int [B], default 0..B-1) key the random
    samples: a pair's result depends only on its own valid matches, its id, the seed and the budget, never on its
    neighbours in the batch or on where its padding lies.

    -> (model [B, 3, 3] float32, inlier_mask [B, K] bool, num_inliers [B] int32).  H is scaled to H[2, 2] = 1, F to
    unit Frobenius norm with its largest-magnitude entry positive.  A pair with fewer valid matches than the minimal
    sample, or with only degenerate samples (e.g. all points collinear), gets a NaN model, an all-false mask and 0.
    return_details=True adds a dict: "best_hypothesis" [B] int32 (the index of the winning hypothesis, -1 when none)
    and "samples" [B, iterations, s] int32 (each hypothesis' sample as ascending columns of K, -1 for a pair below the
    sample size).  No host synchronisation: the call can be captured in a CUDA graph."""
    model, threshold, iterations, seed = check_options(model, threshold, iterations, seed)
    s = SAMPLE_SIZE[model]
    for name, t in (("points0", points0), ("points1", points1)):
        if not torch.is_tensor(t) or t.dtype != torch.float32:
            raise TypeError(f"estimate_geometry: `{name}` must be a float32 tensor (got "
                            f"{t.dtype if torch.is_tensor(t) else type(t).__name__})")
        if not t.is_cuda:
            raise ValueError(f"estimate_geometry: `{name}` must be a CUDA tensor (there is no CPU implementation)")
        if t.dim() != 3 or t.shape[2] != 2:
            raise ValueError(f"estimate_geometry: `{name}` must be [B, K, 2] (got {tuple(t.shape)})")
    if points0.shape != points1.shape:
        raise ValueError(f"estimate_geometry: points0 {tuple(points0.shape)} and points1 {tuple(points1.shape)} differ")
    if points0.device != points1.device:
        raise ValueError(f"estimate_geometry: points0 is on {points0.device}, points1 on {points1.device}")
    dev = points0.device
    B, K = points0.shape[:2]
    if K < s:
        raise ValueError(f"estimate_geometry: K={K} matches per pair is below the {model} sample size {s}")
    if B > 65535:
        raise ValueError(f"estimate_geometry: at most 65535 pairs per call (got {B})")
    mask_in = None
    if valid is not None:
        if not torch.is_tensor(valid):
            raise TypeError("estimate_geometry: `valid` must be None, a bool [B, K] tensor or an integer [B] tensor")
        if valid.device != dev:
            raise ValueError(f"estimate_geometry: `valid` is on {valid.device}, the points on {dev}")
        if valid.dtype == torch.bool:
            if tuple(valid.shape) != (B, K):
                raise ValueError(f"estimate_geometry: a valid mask must be [B, K] = {(B, K)} (got {tuple(valid.shape)})")
            mask_in = valid.contiguous().view(torch.uint8)
        elif valid.dtype in (torch.int32, torch.int64):
            if tuple(valid.shape) != (B,):
                raise ValueError(f"estimate_geometry: valid counts must be [B] = ({B},) (got {tuple(valid.shape)})")
            mask_in = (torch.arange(K, device=dev)[None, :] < valid[:, None]).view(torch.uint8)
        else:
            raise TypeError(f"estimate_geometry: `valid` must be bool or int32 / int64 (got {valid.dtype})")
    ids = None
    if pair_ids is not None:
        if not torch.is_tensor(pair_ids) or pair_ids.dtype not in (torch.int32, torch.int64) \
                or tuple(pair_ids.shape) != (B,) or pair_ids.device != dev:
            raise ValueError(f"estimate_geometry: pair_ids must be an int32 / int64 tensor [B] = ({B},) on {dev}")
        ids = pair_ids.to(torch.int32).contiguous()
    out_model = torch.empty(B, 3, 3, dtype=torch.float32, device=dev)
    out_mask = torch.empty(B, K, dtype=torch.uint8, device=dev)
    out_count = torch.empty(B, dtype=torch.int32, device=dev)
    best = samples = None
    if return_details:
        best = torch.empty(B, dtype=torch.int32, device=dev)
        samples = torch.empty(B, iterations, s, dtype=torch.int32, device=dev)
    if B:
        _lib.require(_lib.GEOMETRY_VERSION, "estimate_geometry")
        lib = _lib.load()
        p0, p1 = points0.contiguous(), points1.contiguous()
        nbytes = lib.lb_geometry_workspace_bytes(B, K, iterations)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(lib.lb_estimate_geometry(p0.data_ptr(), p1.data_ptr(), _lib.ptr(mask_in), _lib.ptr(ids), B, K,
                                            MODELS[model], threshold, iterations, seed, out_model.data_ptr(),
                                            out_mask.data_ptr(), out_count.data_ptr(), _lib.ptr(best),
                                            _lib.ptr(samples), ws.data_ptr(), nbytes, _stream(p0)))
    result = (out_model, out_mask.view(torch.bool), out_count)
    if return_details:
        return result + ({"best_hypothesis": best, "samples": samples},)
    return result


def estimate_on_matches(data, bs, per_pair_bound, options):
    """Runs `estimate_geometry` on a match list as the matcher writes it (mkpts0_f / mkpts1_f [M, 2] with m_bids [M]
    in ascending pair order) and adds data["geom_model"] [bs, 3, 3], data["geom_inliers"] [M] bool (aligned with the
    match list) and data["geom_num_inliers"] [bs] int32.  per_pair_bound: a host bound on any pair's match count."""
    pts0, pts1, bids = data["mkpts0_f"], data["mkpts1_f"], data["m_bids"]
    m = pts0.shape[0]
    dev = pts0.device
    K = max(min(m, per_pair_bound), SAMPLE_SIZE[options["model"]])
    rank = torch.arange(m, device=dev) - torch.searchsorted(bids, bids)   # position of each match within its pair
    p0 = torch.zeros(bs, K, 2, dtype=torch.float32, device=dev)
    p1 = torch.zeros(bs, K, 2, dtype=torch.float32, device=dev)
    valid = torch.zeros(bs, K, dtype=torch.bool, device=dev)
    p0[bids, rank] = pts0.float()
    p1[bids, rank] = pts1.float()
    valid[bids, rank] = True
    model, mask, count = estimate_geometry(p0, p1, valid, **options)
    data.update({"geom_model": model, "geom_inliers": mask[bids, rank], "geom_num_inliers": count})
