"""Every library path on poisoned, guarded memory (tests/poison.py): no output may depend on memory the call did not
write, and no call may write past a buffer it was given.

(a) Each path runs once on ordinary allocations and once under each pattern of `poison.PATTERNS`, with every package
    allocation poisoned and guarded.  Every output must equal the clean run's bit for bit (`util.assert_same`, NaN at
    the same places) and every guard must be intact.  The one exception is what DESIGN.md §11 leaves unspecified: the
    entries of forward_static's capacity buffers at or past min(num_matches, capacity).  Model calls start from an
    empty packed-weight cache, so that the weight packing runs on poisoned memory as well.
(b) The float64 checks of tests/test_kernel_edges_gpu.py and tests/test_guided_gpu.py, run unchanged inside
    poisoned("0xFF") and poisoned("big"): poisoned workspaces must not move a result away from float64.
(c) The same outputs without programmatic dependent launch (LOFTR_B200_PDL=0, in a child process) as with it.

Each case records its paths, patterns, allocations and guard bytes through `util.record`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import loftr_b200
import poison
import test_guided_gpu as GG
import test_kernel_edges_gpu as KE
import util
from cases import BASELINE_CASES, CASES
from loftr_b200 import evaluation, parallel
from match_cap_ref import LIST_KEYS
from poison import poisoned

pytestmark = pytest.mark.gpu
DEV = util.DEV
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_CASE = {c["name"]: c for c in CASES}
# the capacity buffers of forward_static: entries at or past min(num_matches, capacity) are unspecified
STATIC_KEYS = tuple(LIST_KEYS) + ("minside1",)


def _tensors(out):
    """The outputs of a call as a flat dict: tensors and plain values; named tuples and feature banks by field."""
    if hasattr(out, "_asdict"):
        out = out._asdict()
    elif isinstance(out, loftr_b200.ImageFeatures):
        out = {k: getattr(out, k) for k in ("feat_c", "feat_f", "mask", "hw_i", "hw_c", "hw_f")}
    return {k: v for k, v in out.items() if not callable(v)}


def _compare(got, ref, label):
    """got equals ref bit for bit; with a num_matches key, the capacity buffers only below min(count, capacity)."""
    assert set(got) == set(ref), f"{label}: keys {sorted(set(got) ^ set(ref))}"
    live = None
    if "num_matches" in ref:
        util.assert_same(got["num_matches"], ref["num_matches"], label=f"{label}: num_matches")
        live = min(int(ref["num_matches"].item()), ref["b_ids"].shape[0])
    for k, r in ref.items():
        g = got[k]
        if live is not None and k in STATIC_KEYS:
            assert g.shape == r.shape, (label, k)
            g, r = g[:live], r[:live]
        if isinstance(r, dict):
            _compare(g, r, f"{label}: {k}")
        elif isinstance(r, (list, tuple)) and r and torch.is_tensor(r[0]):
            assert len(g) == len(r), (label, k)
            for n, (a, b) in enumerate(zip(g, r)):
                util.assert_same(a, b, label=f"{label}: {k}[{n}]")
        else:
            util.assert_same(g, r, label=f"{label}: {k}")


def _bits(name, run, model=None, patterns=poison.PATTERNS):
    """run() -> outputs, once clean and once under each pattern: the same bits, intact guards.  `model`: its packed
    weights are dropped before every run.  -> the clean outputs."""
    def call():
        if model is not None:
            model.invalidate_packed()
        out = _tensors(run())
        torch.cuda.synchronize()
        return out
    clean = call()
    stats = {"paths": name, "patterns": list(patterns), "keys": len(clean), "allocations": 0, "guard_bytes": 0,
             "poisoned_bytes": 0}
    for p in patterns:
        with poisoned(p) as pz:
            got = call()
        _compare(got, clean, f"{name} [{p}]")
        for k in ("allocations", "guard_bytes", "poisoned_bytes"):
            stats[k] += pz.stats()[k]
    assert stats["allocations"] > 0, f"{name}: nothing was allocated through the package"
    util.record("poisoned_" + name, stats)
    return clean


# ------------------------------------------------------------------------------------------------ (a) forward
FORWARD_CASES = {"ds_thr0": _CASE["ds_thr0"], "ot_thr0_prefilter": dict(_CASE["ot_thr0"], prefilter=True),
                 "ds_masked_scaled": _CASE["ds_masked_scaled"], "ds_unequal": _CASE["ds_unequal"],
                 "ds_empty": _CASE["ds_empty"]}
OPTIONS = ["plain", "full_attention", "match_fp16", "backbone_fp16", "backbone_torch", "conf_matrix", "cap7", "thr-1"]


def _model(case, option="plain"):
    if option == "full_attention":
        case = dict(case, coarse_attention="full", fine_attention="full")
    impl = {"backbone_fp16": "b200_fp16", "backbone_torch": "torch"}.get(option, "auto")
    model, _, _ = util.build_model(case, DEV, impl, "fp16" if option == "match_fp16" else "split")
    cm = model.coarse_matching
    if option == "conf_matrix":
        cm.config["return_conf_matrix"] = True
    elif option == "cap7":
        cm.max_matches_per_pair = 7
    elif option == "thr-1":
        cm.thr = -1.0
    return model


@pytest.mark.parametrize("option", OPTIONS)
@pytest.mark.parametrize("name", list(FORWARD_CASES))
def test_forward_is_bitwise_clean_under_poison(name, option):
    case = FORWARD_CASES[name]
    model = _model(case, option)
    inp = util.device_inputs(case)
    out = _bits(f"forward_{name}_{option}", lambda: util.outputs(util.eager(model, inp)), model)
    if option == "conf_matrix":
        assert "conf_matrix" in out


def test_forward_b8_640x480_is_bitwise_clean_under_poison():
    """Batch 8 at 640 x 480: several column chunks and row tiles per pair in every carved workspace."""
    case = BASELINE_CASES["b8"]
    model = _model(case)
    inp = util.device_inputs(case)
    out = _bits("forward_b8_640x480", lambda: util.outputs(util.eager(model, inp)), model)
    assert out["b_ids"].numel() > 8 * 400


@pytest.mark.parametrize("capacity", ["default", "above_count", "overflow_2"])
def test_forward_static_is_bitwise_clean_under_poison(capacity):
    case = _CASE["ds_thr0"]
    model = _model(case)
    inp = util.device_inputs(case)
    m = util.eager(model, inp)["b_ids"].shape[0]
    assert m > 2
    cap = {"default": None, "above_count": m + 77, "overflow_2": 2}[capacity]

    def run():
        st = dict(inp)
        model.forward_static(st, capacity=cap)
        return util.outputs(st)
    out = _bits(f"forward_static_{capacity}", run, model)
    assert int(out["num_matches"].item()) == m
    assert out["b_ids"].shape[0] == (cap if cap is not None else out["b_ids"].shape[0])


def test_captured_matcher_two_replays_are_bitwise_clean_under_poison():
    """The graph captures the poison fills with the kernels, so every replay poisons its buffers again."""
    case = _CASE["ds_thr0"]
    model = _model(case)
    batches = [util.device_inputs(case, seed) for seed in (1, 2)]

    def run():
        cm = loftr_b200.CapturedMatcher(model, case["n"], case["hw0"], case["hw1"])
        out = {}
        for r, inp in enumerate(batches):
            got = dict(inp)
            cm(got)
            out.update({f"replay{r}_{k}": v for k, v in util.outputs(got).items()})
        return out
    out = _bits("captured_matcher_2_replays", run, model)
    ref = util.outputs(util.eager(model, batches[1]))
    util.assert_same({k: out["replay1_" + k] for k in LIST_KEYS}, ref, LIST_KEYS, "replay vs eager")


# ------------------------------------------------------------------------------------------------ (a) feature banks
BANK = ["repeated_indices", "estimate_fundamental", "estimate_homography", "guide"]


@pytest.mark.parametrize("variant", BANK)
def test_feature_bank_is_bitwise_clean_under_poison(variant):
    case = _CASE["ds_thr0"]
    model = _model(case)
    inp = util.device_inputs(case)
    imgs = torch.cat([inp["image0"], inp["image1"]])           # bank images 0, 1 | 2, 3
    idx0, idx1 = util.idx([0, 1, 0, 1, 0]), util.idx([2, 3, 3, 2, 2])
    opts = {}
    if variant.startswith("estimate_"):
        opts["estimate"] = variant[len("estimate_"):]
    elif variant == "guide":
        opts["guide"] = util.guide("homography", np.repeat(util.H_MODEL[None], 5, 0), 28.0)

    def run():
        bank = model.extract_features(imgs)
        out = {f"bank_{k}": v for k, v in _tensors(bank).items()}
        out.update(model.match_features(bank, idx0, bank, idx1, **opts))
        return out
    out = _bits(f"feature_bank_{variant}", run, model)
    assert out["b_ids"].numel() > 0


# ------------------------------------------------------------------------------------------------ (a) point queries
POINTS = ["image0", "image1", "round_trip", "bank_homography_guide", "bank_fundamental_guide"]


def _query_points(data, side, seed):
    """Every other cell keypoint of image `side`, moved off the grid, with a NaN point and invalid slots."""
    pts = util.grid_points(data, side)[:, ::2].clone()
    rs = np.random.RandomState(seed)
    pts += util.to_dev(rs.uniform(-3.0, 3.0, pts.shape).astype(np.float32))
    pts[0, 1] = float("nan")
    valid = util.to_dev(rs.uniform(size=pts.shape[:2]) > 0.1)
    return pts.contiguous(), valid


@pytest.mark.parametrize("variant", POINTS)
def test_point_queries_are_bitwise_clean_under_poison(variant):
    case = _CASE["ds_masked_scaled"] if variant in ("image0", "image1", "round_trip") else _CASE["ds_thr0"]
    model = _model(case)
    inp = util.device_inputs(case)
    n = case["n"]
    if variant in ("image0", "image1", "round_trip"):
        side = int(variant == "image1")
        pts, valid = _query_points(inp, side, 3 + side)
        args = {"image0": {"points0": pts, "valid0": valid}, "image1": {"points1": pts, "valid1": valid},
                "round_trip": {"points0": pts, "valid0": valid, "round_trip": True}}[variant]

        def call():
            d = dict(inp)
            model.match_points(d, **args)
            return util.outputs(d)
    else:
        kind = variant.split("_")[1]
        imgs = torch.cat([inp["image0"], inp["image1"]])
        i0, i1 = util.idx(list(range(n))), util.idx([n + b for b in range(n)])
        pts, valid = _query_points(inp, 0, 6)
        g = util.guide(kind, np.repeat((util.H_MODEL if kind == "homography" else util.F_MODEL)[None], n, 0), 28.0)

        def call():
            bank = model.extract_features(imgs)
            return model.match_points_features(bank, i0, bank, i1, pts, valid, guide=g)
    out = _bits(f"match_points_{variant}", call, model)
    assert out["qinside"].any()


# ------------------------------------------------------------------------------------------------ (a) guide, rectify
@pytest.mark.parametrize("variant", ["guide", "rectify1", "rectify1_candidates"])
def test_guided_and_rectified_forward_are_bitwise_clean_under_poison(variant):
    case = _CASE["ds_masked_scaled"]
    model = _model(case)
    inp = util.device_inputs(case)
    n, (h, w) = case["n"], case["hw0"]
    extra = {}
    if variant == "guide":
        extra["guide"] = util.guide("fundamental", np.repeat(util.F_MODEL[None], n, 0), 12.0)
    elif variant == "rectify1":
        s0, s1 = util.to_np(inp["scale0"]), util.to_np(inp["scale1"])
        extra["rectify1"] = util.to_dev(np.stack([util.similarity(
            (0.5 * (w - 1) * s0[b, 0], 0.5 * (h - 1) * s0[b, 1]), (0.5 * (w - 1) * s1[b, 0], 0.5 * (h - 1) * s1[b, 1]),
            4.0 + 3 * b, 1.05) for b in range(n)]), torch.float32)
    else:
        size = torch.tensor([[w, h]] * n, device=DEV)
        extra["rectify1_candidates"] = loftr_b200.rotation_candidates(size, size, inp["scale0"], inp["scale1"])
    keys = util.INPUT_KEYS + tuple(extra)
    out = _bits(f"forward_{variant}", lambda: util.outputs(util.eager(model, dict(inp, **extra)), keys), model)
    assert out["b_ids"].numel() > 0


# ------------------------------------------------------------------------------------------------ (a) other entries
def _u8(seed, h, w, c=None):
    rs = np.random.RandomState(seed)
    shape = (h, w) if c is None else (h, w, c)
    return torch.from_numpy(rs.randint(0, 256, shape).astype(np.uint8))


def test_image_front_end_is_bitwise_clean_under_poison():
    """prepare_images / prepare_pairs on ragged lists (device and host images, grey and colour), and warp_images."""
    ragged = [_u8(1, 70, 93).to(DEV), _u8(2, 120, 64, 3), _u8(3, 33, 150).to(DEV)]
    _bits("prepare_images_ragged", lambda: loftr_b200.prepare_images(ragged, resize=96, pad_to="batch"))
    src0 = [_u8(4, 100, 140).to(DEV), _u8(5, 96, 128, 3).to(DEV)]
    src1 = [_u8(6, 80, 60), _u8(7, 130, 90).to(DEV)]
    _bits("prepare_pairs_ragged", lambda: loftr_b200.prepare_pairs(src0, src1, resize=128, pad_to="square",
                                                                   device=DEV))
    img = util.to_dev(np.random.RandomState(8).uniform(size=(3, 1, 56, 72)).astype(np.float32))
    models = util.to_dev(np.stack([util.similarity((36, 28), (30, 25), d, 1.1) for d in (0, 17, -40)]), torch.float32)
    scale = util.to_dev(np.array([[1.0, 1.0], [1.5, 1.25], [0.8, 2.0]], np.float32))
    _bits("warp_images", lambda: {"warped": loftr_b200.warp_images(img, models, (64, 48), scale, scale.flip(1))})


@pytest.mark.parametrize("model_kind", ["homography", "fundamental"])
@pytest.mark.parametrize("K", [255, 256, 257])
def test_geometry_estimator_is_bitwise_clean_under_poison(K, model_kind):
    rs = np.random.RandomState(K)
    B = 5
    p0 = rs.uniform(0, 640, (B, K, 2))
    H = util.H_MODEL.astype(np.float64)
    q = np.concatenate([p0, np.ones((B, K, 1))], 2) @ H.T
    p1 = q[..., :2] / q[..., 2:]
    if model_kind == "fundamental":     # a second plane makes F well posed
        p1[:, ::2] += rs.uniform(-40, 40, (B, (K + 1) // 2, 1)) * np.array([1.0, 0.3])
    p1 += rs.normal(0, 0.3, p1.shape)
    p1[:, ::7] = rs.uniform(0, 640, p1[:, ::7].shape)                      # outliers
    counts = util.to_dev(np.array([K, K - 1, 0, 7, K // 2], np.int32))
    pts0, pts1 = util.to_dev(p0, torch.float32), util.to_dev(p1, torch.float32)

    def run():
        m, mask, n, det = loftr_b200.estimate_geometry(pts0, pts1, counts, model_kind, iterations=64,
                                                        return_details=True)
        return {"model": m, "inliers": mask, "num_inliers": n, **det}
    out = _bits(f"estimate_geometry_{model_kind}_K{K}", run)
    assert int(out["num_inliers"].max()) > 0


def test_epipolar_errors_are_bitwise_clean_under_poison():
    rs = np.random.RandomState(9)
    m, n = 1000, 3
    data = {"mkpts0_f": util.to_dev(rs.uniform(0, 640, (m, 2)).astype(np.float32)),
            "mkpts1_f": util.to_dev(rs.uniform(0, 640, (m, 2)).astype(np.float32)),
            "m_bids": util.to_dev(np.sort(rs.randint(0, n, m)).astype(np.int64)),
            "T_0to1": util.to_dev(np.tile(np.eye(4), (n, 1, 1)) + rs.normal(0, 0.1, (n, 4, 4)), torch.float32),
            "K0": util.to_dev(np.tile(np.diag([500.0, 500, 1]), (n, 1, 1)), torch.float32),
            "K1": util.to_dev(np.tile(np.diag([520.0, 510, 1]), (n, 1, 1)), torch.float32)}

    def run():
        d = dict(data)
        evaluation.compute_symmetrical_epipolar_errors(d)
        return {"epi_errs": d["epi_errs"]}
    _bits("epipolar_errors", run)


def test_pack_unpack_matches_are_bitwise_clean_under_poison():
    cap = 96
    rs = np.random.RandomState(71)
    ranks = []
    for m in (0, cap, 37):
        ranks.append({"mkpts0_f": util.to_dev(rs.uniform(0, 640, (m, 2)).astype(np.float32)),
                      "mkpts1_f": util.to_dev(rs.uniform(0, 640, (m, 2)).astype(np.float32)),
                      "mconf": util.to_dev(rs.uniform(0, 1, m).astype(np.float32)),
                      "m_bids": util.to_dev(np.sort(rs.randint(0, 3, m)).astype(np.int64))})

    def run():
        bufs = [parallel.pack_matches(d, 3 * r, cap) for r, d in enumerate(ranks)]
        out = {f"packed{r}": b[: 1 + ranks[r]["mconf"].shape[0]] for r, b in enumerate(bufs)}   # rows past m: unspecified
        out.update(parallel.unpack_matches(torch.stack(bufs)))
        return out
    out = _bits("pack_unpack_matches", run)
    assert out["counts"] == [0, cap, 37]


# ------------------------------------------------------------------------------------------------ (b) float64
def _param(p):
    return p.values[0] if hasattr(p, "values") else p


CM_POISON = [c for c in KE.CM_SHAPES if c.id in ("L127_S255", "L127_S256", "L127_S257", "L128_S255", "L128_S256",
                                                   "L128_S257", "L129_S255", "L129_S256", "L129_S257",
                                                   "L128_S18915_chunk_clamp", "masks_narrow")]
GUIDED_CASE = [c for c in GG.F64_SHAPES if c.id == "multi_chunk_unequal"][0]


def _f64_cases():
    out = []
    for c in CM_POISON:
        for mt in ("dual_softmax", "sinkhorn"):
            out.append(pytest.param(("cm", c.values[0], mt), id=f"cm_{c.id}_{mt}"))
    for mt in ("dual_softmax", "sinkhorn"):
        out.append(pytest.param(("conf_multi_chunk", mt), id=f"conf_matrix_multi_chunk_{mt}"))
        for kind, radius in (("fundamental", 12.0), ("homography", 28.0)):
            out.append(pytest.param(("guided", mt, kind, radius), id=f"guided_multi_chunk_unequal_{mt}_{kind}"))
    for att in ("linear", "full"):
        out.append(pytest.param(("split_k", att), id=f"tf_split_k_{att}"))
        out.append(pytest.param(("fully_masked", att), id=f"tf_fully_masked_{att}"))
        out.append(pytest.param(("windows", att), id=f"tf_5003_windows_{att}"))
    for W in (3, 5):
        out.append(pytest.param(("fine_pre", W), id=f"fine_preprocess_channel_slice_W{W}"))
        out.append(pytest.param(("fine_match", W), id=f"fine_match_M1_W{W}"))
    return out


def _run_f64(job):
    kind = job[0]
    if kind == "cm":
        KE.test_coarse_matching_shapes_vs_f64(job[1], job[2])
    elif kind == "conf_multi_chunk":
        KE.test_conf_matrix_multi_chunk_vs_f64(job[1])
    elif kind == "guided":
        GG.test_guided_matching_vs_f64(GUIDED_CASE.values[0], *job[1:])
    elif kind == "split_k":
        KE.test_coarse_transformer_split_k_vs_f64(job[1])
    elif kind == "fully_masked":
        KE.test_coarse_transformer_fully_masked_images_vs_f64(job[1])
    elif kind == "windows":
        KE.test_window_transformer_vs_f64(_param([c for c in KE.WINDOWS if c.id == "5003_windows"][0]), job[1])
    elif kind == "fine_pre":
        KE.test_fine_preprocess_vs_f64(job[1], "channel_slice")
    else:
        KE.test_fine_matching_random_vs_f64(job[1], 1)


@pytest.mark.parametrize("pattern", ["0xFF", "big"])
@pytest.mark.parametrize("job", _f64_cases())
def test_float64_checks_hold_under_poison(job, pattern, request):
    """The kernels' float64 rules (match lists by `util.compare_matches`, dense outputs within 4x the fp32 oracle's
    error) with every package allocation poisoned: the references in tests/ allocate normally."""
    with poisoned(pattern) as pz:
        _run_f64(job)
    util.record("poisoned_f64_" + request.node.callspec.id, {"paths": job[0], **pz.stats()})
    assert pz.stats()["allocations"] > 0


# ------------------------------------------------------------------------------------------------ (c) without PDL
_CHILD = r"""
import os, sys
root, path = sys.argv[1], sys.argv[2]
for p in (root, os.path.join(root, "tests"), os.path.join(root, "tests", "golden")):
    sys.path.insert(0, p)
import torch
import test_poisoned_memory_gpu as T
torch.save(T._pdl_outputs(), path)
"""


def _pdl_outputs():
    """forward on ds_thr0 and on the batch-8 640 x 480 case, and forward_static on ds_thr0 -> {label: outputs} on the
    CPU (the live prefix of the static capacity buffers)."""
    res = {}
    for label, case in (("ds_thr0", _CASE["ds_thr0"]), ("b8", BASELINE_CASES["b8"])):
        model = _model(case)
        inp = util.device_inputs(case)
        res[label] = {k: v.cpu() for k, v in util.outputs(util.eager(model, inp)).items() if torch.is_tensor(v)}
        if label == "ds_thr0":
            st = dict(inp)
            model.forward_static(st)
            m = int(st["num_matches"].item())
            res["static_ds_thr0"] = {k: (v[:m] if k in STATIC_KEYS else v).cpu()
                                     for k, v in util.outputs(st).items() if torch.is_tensor(v)}
    return res


def test_outputs_equal_without_programmatic_dependent_launch(tmp_path):
    """The tensor-core kernels launched with PDL (engine.cu launch_persistent) against serialised launches."""
    path = str(tmp_path / "no_pdl.pt")
    env = dict(os.environ, LOFTR_B200_PDL="0")
    proc = subprocess.run([sys.executable, "-c", _CHILD, ROOT, path], env=env, cwd=ROOT, capture_output=True,
                          text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]
    serial = torch.load(path)
    here = _pdl_outputs()
    assert set(serial) == set(here)
    n = 0
    for label, ref in here.items():
        _compare(serial[label], ref, f"LOFTR_B200_PDL=0 {label}")
        n += len(ref)
    assert here["b8"]["b_ids"].numel() > 0
    util.record("pdl_off_vs_on", {"paths": sorted(here), "tensors": n})
