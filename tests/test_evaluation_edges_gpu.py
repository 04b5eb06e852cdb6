"""The epipolar-error kernel against float64, and `evaluate_pairs` (the `test.py` driver) end to end.

epipolar_error_kernel runs through `compute_symmetrical_epipolar_errors`.  Each match is judged by the rule of
tests/epipolar_ref.py, e = |k - r| / (2 |pep| P w + r) against the float64 result r, and the kernel's largest e must
stay within 4x of the fp32 oracle's (or of 2^-24 when that is smaller).  Cases: ScanNet-like indoor pairs, 1600x1200
pairs with |t| from 1e-4 to 1e3, forward motion with matches around the epipole, pure rotation (NaN exactly where
float64 is NaN), unsorted and interleaved m_bids with an empty pair in the middle, ids outside [0, n_pairs) (NaN; 2^32
must not alias pair 0), M at the 256-thread block boundary and 2^21, and the argument forms the wrapper converts
(float64 points, int32 ids, non-contiguous tensors: bit for bit the contiguous float32 call)."""
import os

import numpy as np
import pytest
import torch

import epipolar_ref as R
import util
from metrics_cases import make_scene_batch
from loftr_b200 import evaluation as E

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS = ("mkpts0_f", "mkpts1_f", "m_bids", "T_0to1", "K0", "K1")


def kernel(sc):
    data = {k: torch.from_numpy(np.ascontiguousarray(sc[k])).to(DEV) for k in KEYS}
    E.compute_symmetrical_epipolar_errors(data)
    out = data["epi_errs"].cpu().numpy()
    assert out.dtype == np.float32 and out.shape == (len(sc["m_bids"]),)
    return out


def check_rule(sc, name):
    k = kernel(sc)
    r, scale = R.terms(sc)
    with np.errstate(all="ignore"):
        o = R.oracle32(sc)
    nan = np.isnan(r)
    assert np.array_equal(np.isnan(k), nan), (name, int(np.isnan(k).sum()), int(nan.sum()))
    assert np.isfinite(k[~nan]).all(), name
    stats = {"M": len(k), "nan": int(nan.sum())}
    if (~nan).any():
        ek, eo = np.nanmax(R.rule_error(k, r, scale)), np.nanmax(R.rule_error(o[~nan], r[~nan], scale[~nan]))
        bound = 4 * max(eo, R.ULP)
        stats.update(max_e_kernel_ulp=ek / R.ULP, max_e_oracle_ulp=eo / R.ULP, bound_ulp=bound / R.ULP)
        assert ek <= bound, (name, ek / R.ULP, eo / R.ULP)
    util.record(f"epipolar_{name}", stats)
    return k


@pytest.mark.parametrize("seed", [0, 1, 7])
def test_indoor_pairs(seed):
    check_rule(make_scene_batch(seed, 3), f"indoor_seed{seed}")


def test_outdoor_translation_magnitudes():
    check_rule(R.outdoor_scene(3), "outdoor_t_1e-4_to_1e3")


def test_forward_motion_near_the_epipole():
    check_rule(R.forward_scene(4), "forward_motion")


def test_pure_rotation_is_nan():
    k = check_rule(R.rotation_scene(5), "pure_rotation")
    assert np.isnan(k[:200]).all() and np.isfinite(k[200:]).all()


def test_unsorted_interleaved_ids_with_an_empty_pair():
    sc = make_scene_batch(11, 5)
    keep = sc["m_bids"] != 2                         # pair 2 keeps its pose but has no match
    perm = np.random.RandomState(0).permutation(int(keep.sum()))
    sc = {k: (v[keep][perm] if k in ("mkpts0_f", "mkpts1_f", "m_bids") else v) for k, v in sc.items()}
    assert (np.diff(sc["m_bids"]) < 0).any()
    k = check_rule(sc, "unsorted_ids_empty_pair")
    # each match keeps the value it has in its own pair's sorted call
    for b in (0, 4):
        sel = sc["m_bids"] == b
        one = {"mkpts0_f": sc["mkpts0_f"][sel], "mkpts1_f": sc["mkpts1_f"][sel], "m_bids": np.zeros(sel.sum(), np.int64),
               "T_0to1": sc["T_0to1"][b:b + 1], "K0": sc["K0"][b:b + 1], "K1": sc["K1"][b:b + 1]}
        assert np.array_equal(kernel(one).view(np.uint32), k[sel].view(np.uint32)), b


def test_ids_outside_the_pairs_are_nan():
    sc = make_scene_batch(12, 3)
    n = len(sc["m_bids"])
    bad = np.random.RandomState(1).permutation(n)[:30]
    bids = sc["m_bids"].copy()
    bids[bad[:10]], bids[bad[10:20]], bids[bad[20:]] = -1, 3, 2 ** 32    # 2^32 is pair 0 in its low 32 bits
    k = check_rule(dict(sc, m_bids=bids), "ids_outside_pairs")
    assert np.isnan(k[bad]).all() and np.isfinite(np.delete(k, bad)).all()


@pytest.mark.parametrize("M", [1, 255, 256, 257, 2 ** 21])
def test_block_boundaries(M):
    check_rule(R.sized_scene(M % 1000, M), f"M{M}")


def test_argument_forms_are_bitwise_the_float32_call():
    sc = make_scene_batch(13, 4)
    want = kernel(sc)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in sc.items()}
    # float64 points and poses, int32 ids
    d = {"mkpts0_f": t["mkpts0_f"].double(), "mkpts1_f": t["mkpts1_f"].double(), "m_bids": t["m_bids"].int(),
         "T_0to1": t["T_0to1"].double(), "K0": t["K0"].double(), "K1": t["K1"].double()}
    E.compute_symmetrical_epipolar_errors(d)
    assert np.array_equal(d["epi_errs"].cpu().numpy().view(np.uint32), want.view(np.uint32))
    # non-contiguous views of every input
    wide = lambda x: torch.stack([x, torch.full_like(x, 7)], -1)[..., 0]
    nc = {k: wide(v) for k, v in t.items()}
    nc["mkpts0_f"] = torch.cat([t["mkpts0_f"], t["mkpts0_f"]], 1)[:, :2]
    nc["K1"] = t["K1"].transpose(1, 2).contiguous().transpose(1, 2)
    assert not any(v.is_contiguous() for v in nc.values())
    E.compute_symmetrical_epipolar_errors(nc)
    assert np.array_equal(nc["epi_errs"].cpu().numpy().view(np.uint32), want.view(np.uint32))
    util.record("epipolar_argument_forms", {"M": len(want), "bitwise": 1})


# ------------------------------------------------------------------------------------------------ evaluate_pairs
def _write_dataset(root, rs):
    """Five ScanNet-style pairs over two scenes (images, cam-to-world poses, test.npz, intrinsics.npz); the last pair
    repeats the second."""
    import cv2
    names = [(707, 0, 15, 585), (707, 0, 30, 45), (708, 1, 0, 90), (708, 1, 15, 105), (707, 0, 30, 45)]
    K = {"scene0707_00": np.array([[577.0, 0, 319.5], [0, 578.0, 239.5], [0, 0, 1]]),
         "scene0708_01": np.array([[580.0, 0, 320.0], [0, 581.0, 240.0], [0, 0, 1]])}
    c2w = {}
    for scene, sub, *frames in names:
        d = f"scene{scene:04d}_{sub:02d}"
        for fr in frames:
            if (d, fr) in c2w:
                continue
            img = cv2.resize((rs.rand(60, 80) * 255).astype(np.uint8), (640, 480), interpolation=cv2.INTER_CUBIC)
            os.makedirs(os.path.join(root, d, "color"), exist_ok=True)
            os.makedirs(os.path.join(root, d, "pose"), exist_ok=True)
            with open(os.path.join(root, d, "color", f"{fr}.jpg"), "wb") as f:
                f.write(cv2.imencode(".png", img)[1].tobytes())      # cv2.imread reads by content
            pose = np.eye(4)
            pose[:3, :3], pose[:3, 3] = R._rot(rs, 0.3), rs.standard_normal(3)
            c2w[(d, fr)] = pose
            np.savetxt(os.path.join(root, d, "pose", f"{fr}.txt"), pose, fmt="%.17g", delimiter=" ")
    np.savez(os.path.join(root, "intrinsics.npz"), **K)
    return np.array(names, np.uint16), c2w


def test_evaluate_pairs_end_to_end(tmp_path):
    rs = np.random.RandomState(3)
    root = str(tmp_path)
    names, c2w = _write_dataset(root, rs)
    rel = np.zeros((len(names), 12), np.float32)
    np.savez(os.path.join(root, "test.npz"), name=names, rel_pose=rel)
    pairs = E.load_scannet_pair_list(os.path.join(root, "test.npz"), os.path.join(root, "intrinsics.npz"))
    # the pose files give T_0to1 = w2c_1 w2c_0^-1 (ScanNet stores cam-to-world)
    for i, p in enumerate(pairs):
        T = E._rel_pose_from_files(root, p["pose_names"])
        d = p["scene_id"]
        want = np.linalg.inv(c2w[(d, int(names[i][3]))]) @ c2w[(d, int(names[i][2]))]
        assert T.dtype == np.float32
        np.testing.assert_allclose(T, want, rtol=1e-6, atol=1e-6)
        rel[i] = T[:3].reshape(-1)
    np.savez(os.path.join(root, "test.npz"), name=names, rel_pose=rel)
    pairs = E.load_scannet_pair_list(os.path.join(root, "test.npz"), os.path.join(root, "intrinsics.npz"))
    case = {"name": "evaluate_pairs", "n": 2, "hw0": (480, 640), "hw1": (480, 640), "thr": 0.0, "images": "smooth"}
    model, _, _ = util.build_model(case, DEV)
    import cv2
    cv2.setRNGSeed(0)           # OpenCV's RANSAC draws from its global RNG
    agg, metrics = E.evaluate_pairs(model, pairs, root, batch_size=2, device=DEV)
    assert metrics["identifiers"][0] == "scene0707_00/color/15.jpg#scene0707_00/color/585.jpg"
    assert metrics["identifiers"] == ["#".join(p["pair_names"]) for p in pairs]
    assert metrics["identifiers"][1] == metrics["identifiers"][4]
    assert len(metrics["epi_errs"]) == len(metrics["R_errs"]) == len(metrics["t_errs"]) == 5
    assert agg == E.aggregate_metrics(metrics)
    # every pair's errors are its slice of the batch the driver ran (batches of 2: the last one holds one pair)
    for lo in range(0, 5, 2):
        chunk = pairs[lo:lo + 2]
        batch = {k: torch.stack([E._read_gray(os.path.join(root, p["pair_names"][j])) for p in chunk]).to(DEV)
                 for j, k in enumerate(("image0", "image1"))}
        batch["T_0to1"] = torch.from_numpy(np.stack([E._rel_pose_from_files(root, p["pose_names"]) for p in chunk])).to(DEV)
        batch["K0"] = batch["K1"] = torch.from_numpy(np.stack([p["K"] for p in chunk])).to(DEV)
        model(batch)
        E.compute_symmetrical_epipolar_errors(batch)
        bids, epi = batch["m_bids"].cpu().numpy(), batch["epi_errs"].cpu().numpy()
        for b in range(len(chunk)):
            assert np.array_equal(metrics["epi_errs"][lo + b].view(np.uint32), epi[bids == b].view(np.uint32)), lo + b
    assert sum(len(e) for e in metrics["epi_errs"]) > 0
    # the pair list's rel_pose column carries the same T: the same metrics
    cv2.setRNGSeed(0)
    agg2, metrics2 = E.evaluate_pairs(model, pairs, root, batch_size=2, device=DEV, rel_pose_from_list=True)
    assert agg2 == agg and metrics2["identifiers"] == metrics["identifiers"]
    assert metrics2["R_errs"] == metrics["R_errs"] and metrics2["t_errs"] == metrics["t_errs"]
    for a, b in zip(metrics["epi_errs"], metrics2["epi_errs"]):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    util.record("evaluate_pairs", {"pairs": 5, "matches": sum(len(e) for e in metrics["epi_errs"]), **agg})
