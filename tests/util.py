"""Shared helpers of the parity tests: the model with the test weights, the numpy oracle's forward (whole batch and per
pair, cached), the match-list rule, the GPU matcher harness (device inputs, eager forward, static = eager, bitwise
comparison, query points, guides and homographies) and the fake libraries of the binding tests."""
from __future__ import annotations

import math
import os

import numpy as np
import torch

import weights as W
from cases import build_cfg, build_cm_inputs, build_inputs  # noqa: F401
from match_cap_ref import LIST_KEYS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda:0"


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def build_model(case, device="cpu", backbone_impl="auto", match_precision="split"):
    """loftr_b200.LoFTR with the case's configuration (attention kinds included), the deterministic RandomState weights
    of tests/golden/weights.py and TF32 off (torch's fp32 products stay fp32) -> (model on `device`, cfg, state)."""
    import loftr_b200
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = build_cfg(case)
    model = loftr_b200.LoFTR(cfg, backbone_impl=backbone_impl, match_precision=match_precision).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    state = W.make_state(shapes, seed=case.get("wseed", 0))
    if "bin_score" in case and "coarse_matching.bin_score" in state:
        state["coarse_matching.bin_score"] = np.asarray(case["bin_score"], np.float32)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    return model.to(device), cfg, state


def device_inputs(case, seed=None):
    """The case's input batch (image seed `seed` instead of the case's) as tensors on the GPU"""
    if seed is not None:
        case = dict(case, iseed=seed)
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in build_inputs(case).items()}


def eager(model, inp):
    """model(batch) on a copy of `inp` -> the batch dict with every output"""
    data = dict(inp)
    model(data)
    return data


def assert_static_equals_eager(st, eager, label):
    """The live prefix of every list output of forward_static / CapturedMatcher equals the eager forward bit for bit,
    with the eager dtypes and sizes, within the capacity, and mkpts0_f aliases mkpts0_c as in the eager forward."""
    m = int(st["num_matches"].item())
    assert m == eager["b_ids"].shape[0], f"{label}: count {m} vs eager {eager['b_ids'].shape[0]}"
    assert m <= st["b_ids"].shape[0]
    for k in LIST_KEYS:
        assert st[k].dtype == eager[k].dtype, (label, k)
        assert torch.equal(st[k][:m], eager[k]), f"{label}: {k} differs from the eager forward"
    assert st["mkpts0_f"] is st["mkpts0_c"]
    for k in ("bs", "hw0_i", "hw1_i", "hw0_c", "hw1_c", "hw0_f", "hw1_f", "W"):
        assert st[k] == eager[k], (label, k)


INPUT_KEYS = ("image0", "image1", "mask0", "mask1", "scale0", "scale1")
# models in output coordinates (image pixels; source pixels with scales): x1 ~ H x0, and F = [e']_x H
H_MODEL = np.array([[1.03, 0.04, 6.0], [-0.03, 0.97, -5.0], [2e-5, -1e-5, 1.0]], np.float32)
_E1 = np.array([140.0, 60.0, 1.0])
F_MODEL = (np.array([[0, -_E1[2], _E1[1]], [_E1[2], 0, -_E1[0]], [-_E1[1], _E1[0], 0]]) @ H_MODEL).astype(np.float32)
F_MODEL /= np.abs(F_MODEL).max()


def inputs(data):
    """The forward inputs of a batch dict."""
    return {k: v for k, v in data.items() if k in INPUT_KEYS}


def outputs(data, keys=INPUT_KEYS):
    """The entries of a batch dict that are not inputs (`keys`): what a call wrote."""
    return {k: v for k, v in data.items() if k not in keys}


def same(got, ref, nan_equal=True):
    """Bitwise equality of two outputs: the same dtype and shape, NaN at the same places (with `nan_equal`; without it
    a NaN is unequal to everything, as in torch.equal) and every other value equal, compared without any cast.
    Non-tensors compare with ==."""
    if not torch.is_tensor(ref):
        return got == ref
    if not torch.is_tensor(got) or got.dtype != ref.dtype or got.shape != ref.shape:
        return False
    if nan_equal and ref.is_floating_point():
        ng, nr = torch.isnan(got), torch.isnan(ref)
        return torch.equal(ng, nr) and torch.equal(got[~ng], ref[~nr])
    return torch.equal(got, ref)


def assert_same(got, ref, keys=None, label="", nan_equal=True):
    """`same` for two outputs, or for the entries `keys` (default: every key of `ref`) of two output dicts."""
    if not isinstance(ref, dict):
        assert same(got, ref, nan_equal), f"{label} differs"
        return
    for k in ref if keys is None else keys:
        assert same(got[k], ref[k], nan_equal), f"{label}: {k} differs"


def to_dev(x, dtype=None):
    """array -> tensor on the GPU (in `dtype`, or the array's own)"""
    t = torch.as_tensor(np.ascontiguousarray(x))
    return t.to(DEV) if dtype is None else t.to(DEV, dtype)


def to_np(t):
    return t.detach().cpu().numpy()


def idx(v):
    """int64 image indices on the GPU"""
    return torch.tensor(v, dtype=torch.int64, device=DEV)


def frames(case):
    """The case's images, masks and scales as one set of 2n frames (image0 of every pair, then image1)."""
    d = device_inputs(case)
    cat = lambda k: torch.cat([d[k + "0"], d[k + "1"]]) if k + "0" in d else None
    return cat("image"), cat("mask"), cat("scale")


def grid_points(data, side=0):
    """Every cell keypoint of image `side` in source pixels, as the forward computes mkpts{side}_c -> [N, cells, 2]."""
    n, _, h, w = data[f"image{side}"].shape
    return bank_grid_points(torch.arange(n, device=DEV), (h // 8, w // 8), data.get(f"scale{side}"))


def bank_grid_points(ids, hw_c, scales=None):
    """`grid_points` of the bank images `ids`, whose scales are scales[ids] -> [len(ids), cells, 2]."""
    hc, wc = hw_c
    i = torch.arange(hc * wc, device=DEV)
    cell = torch.stack([i % wc, i // wc], 1).float()[None].expand(len(ids), -1, -1)
    s = torch.full((len(ids), 1, 2), 8.0, device=DEV) if scales is None else 8.0 * scales[ids][:, None, :]
    return (cell * s).contiguous()


def guide(kind, model, radius):
    """A guide dict: kind "homography" | "fundamental", model [N, 3, 3] (cast to float32), radius in pixels."""
    return {"kind": kind, "model": to_dev(np.asarray(model, np.float32)), "radius": radius}


def similarity(c0, c1, deg, zoom, persp=(0.0, 0.0)):
    """x1 = c1 + zoom R(deg) (x0 - c0), with a perspective row (persp, 1) in the centred frame, as a float64 [3, 3]."""
    a = math.radians(deg)
    t0 = np.array([[1, 0, -c0[0]], [0, 1, -c0[1]], [0, 0, 1]])
    t1 = np.array([[1, 0, c1[0]], [0, 1, c1[1]], [0, 0, 1]])
    r = np.array([[zoom * math.cos(a), -zoom * math.sin(a), 0], [zoom * math.sin(a), zoom * math.cos(a), 0],
                  [persp[0], persp[1], 1]])
    return t1 @ r @ t0


# ------------------------------------------------------------------------------------------------ fake libraries
def old_library(monkeypatch, version):
    """`_lib.load()` returns a library that reports `version` and exports nothing else."""
    from loftr_b200 import _lib

    class OldLib:
        def lb_version(self):
            return version

    monkeypatch.setattr(_lib, "load", lambda: OldLib())


def load_without(monkeypatch, names, version=110):
    """`_lib.load()` on what ctypes.CDLL gives for a build of `version` that exports every declared symbol but `names`
    -> the loaded library."""
    from loftr_b200 import _lib

    class Exports:
        def __init__(self):
            for n in _lib.SIGNATURES:
                if n not in names:
                    setattr(self, n, type("Fn", (), {})())
            self.lb_version = lambda: version

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib.C, "CDLL", lambda path: Exports())
    monkeypatch.setattr(_lib.os.path, "exists", lambda path: True)
    return _lib.load()


def host_bank(model, k=3, masks=False):
    """A host bank of k 96x128 images tied to the model's current weights (never matched: nothing here launches)."""
    from loftr_b200.loftr import ImageFeatures
    mask = torch.ones(k, 12, 16, dtype=torch.bool) if masks else None
    return ImageFeatures(torch.zeros(k, 256, 12, 16), torch.zeros(k, 128, 48, 64), mask, torch.Size((96, 128)),
                         torch.Size((12, 16)), torch.Size((48, 64)), model._bank_key())


def stages_unreachable(monkeypatch, model):
    """The model's matching stages raise if reached, so that a test sees validation stop a call before them -> model"""
    def reached(*a, **k):
        raise AssertionError("a matching stage was reached")
    for name in ("_match_points", "_coarse_tokens", "_backbone", "_backbone_pairs"):
        monkeypatch.setattr(model, name, reached)
    return model


def _backbone(model, i0, i1):
    """PyTorch backbone of one batch (both images in one pass when their sizes agree) -> c0, c1, f0, f1 float32 numpy"""
    with torch.no_grad():
        if i0.shape == i1.shape:
            fc, ff = model.backbone(torch.cat([i0, i1], 0))
            (c0, c1), (f0, f1) = fc.split(i0.shape[0]), ff.split(i0.shape[0])
        else:
            (c0, f0), (c1, f1) = model.backbone(i0), model.backbone(i1)
    return [t.float().cpu().numpy() for t in (c0, c1, f0, f1)]


def oracle_forward(case, backbone_device="cpu"):
    """PyTorch backbone (the part that stays PyTorch) + numpy oracle for everything after it."""
    from oracle import loftr_oracle as O
    model, cfg, state = build_model(case, backbone_device)
    inp = build_inputs(case)
    c0, c1, f0, f1 = _backbone(model, *(torch.from_numpy(inp[k]).to(backbone_device) for k in ("image0", "image1")))
    return O.hot_path(c0, c1, f0, f1, state, cfg, inp["image0"].shape[2:], inp["image1"].shape[2:],
                      inp.get("mask0"), inp.get("mask1"), inp.get("scale0"), inp.get("scale1"))


def near_tie_top2_f64(x0, x1, mc_cfg, m0=None, m1=None, block=2048):
    """fp64 dual-softmax confidence of ONE pair from coarse features x0 [L, C], x1 [S, C] (row-blocked, so that
    L = S = 19200 needs ~1 GB): the two largest confidences of every row and of every column -- the statistics
    `compare_matches` uses to adjudicate non-shared matches as near-ties (SURVEY.md §7 hard part 2;
    reference coarse_matching.py:106-119 evaluated in float64)."""
    c = x0.shape[1]
    a = x0.astype(np.float64) / np.sqrt(c)
    b = x1.astype(np.float64) / np.sqrt(c)
    temp = float(mc_cfg["dsmax_temperature"])
    L, S = a.shape[0], b.shape[0]

    def sim_block(lo, hi):
        s = (a[lo:hi] @ b.T) / temp
        if m0 is not None:
            s[~(m0[lo:hi, None] & m1[None, :])] = -1e9
        return s

    row_lse = np.empty(L)
    col_m = np.full(S, -np.inf)
    col_l = np.zeros(S)
    for lo in range(0, L, block):
        s = sim_block(lo, min(lo + block, L))
        m = s.max(1)
        row_lse[lo:lo + block] = m + np.log(np.exp(s - m[:, None]).sum(1))
        bm = s.max(0)
        nm = np.maximum(col_m, bm)
        col_l = col_l * np.exp(col_m - nm) + np.exp(s - nm[None, :]).sum(0)
        col_m = nm
    col_lse = col_m + np.log(col_l)
    row_top2 = np.empty((L, 2))
    col_top2 = np.zeros((S, 2))
    for lo in range(0, L, block):
        hi = min(lo + block, L)
        conf = np.exp(2 * sim_block(lo, hi) - row_lse[lo:hi, None] - col_lse[None, :])
        row_top2[lo:hi] = -np.sort(-np.partition(conf, S - 2, axis=1)[:, S - 2:], axis=1)
        k = conf.shape[0]
        blk = np.partition(conf, k - 2, axis=0)[k - 2:] if k >= 2 else np.vstack([conf, np.zeros_like(conf)])
        col_top2 = -np.sort(-np.concatenate([col_top2, blk.T], axis=1), axis=1)[:, :2]
    return row_top2, col_top2


CACHE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_oracle_cache")


def _cache_key(case, adjudicate):
    """Hash of the case and of every source file the oracle result depends on."""
    import hashlib
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    h = hashlib.sha1(json.dumps([case, bool(adjudicate)], sort_keys=True, default=str).encode())
    for rel in ("oracle/loftr_oracle.py", "tests/util.py", "tests/golden/weights.py", "tests/golden/cases.py",
                "tests/golden/full_cases.py", "loftr_b200/backbone.py", "loftr_b200/config.py"):
        h.update(open(os.path.join(root, rel), "rb").read())
    return h.hexdigest()[:20]


def oracle_forward_per_pair(case, backbone_device="cpu", adjudicate=True, use_cache=True):
    """Cached front of `_oracle_forward_per_pair`: the oracle is pure CPU work, so its result for a (case, sources)
    key may be precomputed (tools/precompute_oracle.py) into tests/_oracle_cache/ (git-ignored; a missing or stale
    entry is simply recomputed here)."""
    path = os.path.join(CACHE, f"{case.get('name', 'case')}_{_cache_key(case, adjudicate)}.npz")
    if use_cache and os.path.exists(path):
        z = dict(np.load(path))
        gold = {k: z.pop(k) for k in ("row_top2_f64", "col_top2_f64") if k in z} or None
        return z, gold
    res, gold = _oracle_forward_per_pair(case, backbone_device, adjudicate)
    if use_cache:
        try:
            os.makedirs(CACHE, exist_ok=True)
            np.savez(path + ".tmp.npz", **res, **(gold or {}))
            os.replace(path + ".tmp.npz", path)
        except OSError:
            pass
    return res, gold


def _oracle_forward_per_pair(case, backbone_device="cpu", adjudicate=True):
    """`oracle_forward` for a whole batch: the PyTorch backbone runs once on `backbone_device`, the numpy oracle
    then processes ONE PAIR AT A TIME (pairs are independent end to end, reference loftr.py:29-75; this bounds the
    L x S temporaries to one pair) and the per-pair lists are concatenated in (b, i) order.  With `adjudicate`
    (dual-softmax) the fp64 near-tie statistics of every pair are returned as row_top2_f64 / col_top2_f64."""
    from oracle import loftr_oracle as O
    model, cfg, state = build_model(case, backbone_device)
    inp = build_inputs(case)
    feats = [_backbone(model, *(torch.from_numpy(inp[k][b:b + 1]).to(backbone_device) for k in ("image0", "image1")))
             for b in range(inp["image0"].shape[0])]
    keys = ["b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f"]
    parts = {k: [] for k in keys}
    rows, cols, fc0 = [], [], []
    opt = lambda name, b: inp[name][b:b + 1] if name in inp else None
    for b, (c0, c1, f0, f1) in enumerate(feats):
        out = O.hot_path(c0, c1, f0, f1, state, cfg, inp["image0"].shape[2:], inp["image1"].shape[2:],
                         opt("mask0", b), opt("mask1", b), opt("scale0", b), opt("scale1", b))
        for k in keys:
            parts[k].append(out[k] + b if k == "b_ids" else out[k])
        fc0.append(out["feat_c0"][:, ::4])      # every 4th token row: keeps the cache small, still position-sensitive
        if adjudicate and cfg["match_coarse"]["match_type"] == "dual_softmax":
            m0 = inp["mask0"][b].reshape(-1) if "mask0" in inp else None
            m1 = inp["mask1"][b].reshape(-1) if "mask1" in inp else None
            r, c = near_tie_top2_f64(out["feat_c0"][0], out["feat_c1"][0], cfg["match_coarse"], m0, m1)
            rows.append(r)
            cols.append(c)
    res = {k: np.concatenate(v, 0) for k, v in parts.items()}
    res["feat_c0_s4"] = np.concatenate(fc0, 0)
    gold = {"row_top2_f64": np.stack(rows), "col_top2_f64": np.stack(cols)} if rows else None
    return res, gold


def match_keys(b, i, j):
    return {(int(x), int(y), int(z)) for x, y, z in zip(b, i, j)}


def compare_matches(got, ref, gold=None, conf_rtol=1e-3, px_tol=0.5, min_overlap=0.995, label=""):
    """Compare two match lists by (b, i, j) key (SURVEY.md §7 hard part 2).

    - the key sets must overlap >= min_overlap (relative to the larger set);
    - every non-shared match must be a near-tie / near-threshold case according to the fp64 reference
      statistics in `gold` (row_top2_f64 / col_top2_f64) when they are available;
    - on the intersection: mconf within rtol, keypoints within px_tol pixels.
    """
    kg = {k: n for n, k in enumerate(zip(got["b_ids"].tolist(), got["i_ids"].tolist(), got["j_ids"].tolist()))}
    kr = {k: n for n, k in enumerate(zip(ref["b_ids"].tolist(), ref["i_ids"].tolist(), ref["j_ids"].tolist()))}
    common = sorted(set(kg) & set(kr))
    big = max(len(kg), len(kr))
    if big == 0:
        return {"n": 0, "overlap": 1.0}
    overlap = len(common) / big
    adjudicated = gold is not None and "row_top2_f64" in gold
    # a single adjudicated near-tie flip is always tolerated (on a 150-match golden it alone is 0.7 %)
    assert overlap >= min_overlap or (adjudicated and big - len(common) <= 1), \
        f"{label}: match-set overlap {overlap:.4f} ({len(kg)} vs {len(kr)} matches)"
    n_ties = 0
    if adjudicated:
        for (b, i, j) in set(kg) ^ set(kr):
            r, c = gold["row_top2_f64"][b, i], gold["col_top2_f64"][b, j]
            tie = min(abs(r[0] - r[1]) / max(r[0], 1e-30), abs(c[0] - c[1]) / max(c[0], 1e-30))
            assert tie < 1e-2, f"{label}: match {(b, i, j)} differs and is not a near-tie (gap {tie:.3e})"
            n_ties += 1
    ig = np.array([kg[k] for k in common])
    ir = np.array([kr[k] for k in common])
    stats = {"n": len(common), "overlap": overlap, "n_got": len(kg), "n_ref": len(kr),
             "non_shared_adjudicated_near_ties": n_ties if adjudicated else None}
    # the list order must be ascending (b, i) like torch.where
    order = [k[:2] for k in sorted(kg, key=kg.get)]
    assert order == sorted(order), f"{label}: match list is not ordered by (b, i)"
    for key, tol in (("mconf", None), ("mkpts0_c", px_tol), ("mkpts1_c", px_tol), ("mkpts0_f", px_tol),
                     ("mkpts1_f", px_tol)):
        if key not in got or key not in ref:
            continue
        g, r = np.asarray(got[key])[ig], np.asarray(ref[key])[ir]
        if key == "mconf":
            rel = np.abs(g - r) / np.maximum(np.abs(r), 1e-30)
            stats["mconf_rel_max"] = float(rel.max())
            assert rel.max() <= conf_rtol, f"{label}: mconf rel err {rel.max():.3e} > {conf_rtol}"
        else:
            d = np.abs(g - r).max() if len(g) else 0.0
            stats[key + "_max"] = float(d)
            assert d < tol, f"{label}: {key} differs by {d:.4f} px"
    return stats


def record(name, stats):
    """Append parity statistics to gpurun_out/parity_stats.jsonl (kept as evidence; prints are captured by pytest)."""
    import json
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "parity_stats.jsonl"), "a") as f:
            f.write(json.dumps({"test": name, **{k: (float(v) if isinstance(v, (int, float)) else v) for k, v in stats.items()}}) + "\n")
    except OSError:
        pass
