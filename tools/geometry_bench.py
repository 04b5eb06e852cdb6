"""Two-view geometry estimator (`loftr_b200.estimate_geometry`) against the matcher call it follows.

Workloads: B in {1, 8, 32} pairs x K in {512, 2048} matches per pair x {homography, fundamental}, synthetic scenes from
a fixed seed with 30 % outliers, the default budget of 2048 hypotheses and a 3 px threshold.  Per workload:
  estimator     CUDA events around one `estimate_geometry` call (all three launches and the host glue), after warm-up;
  matcher       CUDA events around one `match_features` call on B pairs of 640x480 images (random-weight model, features
                extracted once, match_coarse.max_matches_per_pair = K, so the pairs carry at most K matches each);
  opencv        host clock around cv2.findHomography / cv2.findFundamentalMat (RANSAC, 3 px, 2048 iterations) over
                the B pairs one after the other, on host arrays; absent when cv2 cannot be imported.
Reported: ms (min / median / max over --steps), the estimator's share of the matcher's median, the GPU name and power
limit.  Prints one JSON line per workload; fails without a CUDA device.

    python tools/geometry_bench.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import loftr_b200  # noqa: E402
from measure import alternate, gpu_label, require_gpu, stats  # noqa: E402

BATCHES = (1, 8, 32)
KS = (512, 2048)
MODELS = ("homography", "fundamental")
ITERATIONS, THRESHOLD = 2048, 3.0


def scenes(rs, model, B, K, outliers=0.3):
    """[B, K, 2] float32 pairs: a random homography, or a random calibrated two-view setup, 0.5 px noise."""
    p0 = rs.uniform((0, 0), (640, 480), (B, K, 2))
    p1 = np.empty_like(p0)
    for b in range(B):
        if model == "homography":
            h = np.eye(3) + np.diag(rs.uniform(-.1, .1, 3)) * [1, 1, 0]
            h[:2, 2], h[2, :2] = rs.uniform(-40, 40, 2), rs.uniform(-2e-4, 2e-4, 2)
            q = p0[b] @ h[:, :2].T + h[:, 2]
            p1[b] = q[:, :2] / q[:, 2:]
        else:
            kk = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
            depth = rs.uniform(6, 14, K)
            X = np.linalg.solve(kk, np.concatenate([p0[b], np.ones((K, 1))], 1).T).T * depth[:, None]
            x1 = (X + [1.0, 0.1, 0.2]) @ kk.T
            p1[b] = x1[:, :2] / x1[:, 2:]
    p1 += 0.5 * rs.standard_normal(p1.shape)
    out = rs.uniform(0, 1, (B, K)) < outliers
    p1[out] = rs.uniform((0, 0), (640, 480), (int(out.sum()), 2))
    return p0.astype(np.float32), p1.astype(np.float32)


def matcher():
    import weights as W
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict({k: torch.from_numpy(v) for k, v in W.make_state(shapes, seed=0).items()})
    model = model.cuda()
    g = torch.Generator().manual_seed(0)
    imgs = torch.nn.functional.interpolate(torch.rand(2 * max(BATCHES), 1, 120, 160, generator=g), size=(480, 640),
                                           mode="bilinear", align_corners=False).cuda()
    return model, model.extract_features(imgs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    require_gpu("geometry_bench")
    try:
        import cv2
    except ImportError:
        cv2 = None
    info = gpu_label()
    model, bank = matcher()
    rs = np.random.RandomState(0)
    for B in BATCHES:
        i0 = torch.arange(0, 2 * B, 2, device="cuda")
        i1 = i0 + 1
        for K in KS:
            model.coarse_matching.max_matches_per_pair = K
            out = model.match_features(bank, i0, bank, i1)
            per_pair = torch.bincount(out["m_bids"], minlength=B).float().mean().item()
            t_match = alternate({"matcher": lambda: model.match_features(bank, i0, bank, i1)}, args.steps, args.warmup,
                                flush=False)[0]["matcher"]
            for name in MODELS:
                a0, a1 = scenes(rs, name, B, K)
                p0, p1 = torch.from_numpy(a0).cuda(), torch.from_numpy(a1).cuda()
                t_est = alternate({"estimator": lambda: loftr_b200.estimate_geometry(
                    p0, p1, model=name, threshold=THRESHOLD, iterations=ITERATIONS)}, args.steps, args.warmup,
                    flush=False)[0]["estimator"]
                row = {"workload": f"B{B}_K{K}_{name}", "B": B, "K": K, "model": name, "iterations": ITERATIONS,
                       "estimator_ms": stats(t_est), "matcher_ms": stats(t_match),
                       "matcher_matches_per_pair": round(per_pair, 1),
                       "estimator_share_of_matcher": round(stats(t_est)["median"] / stats(t_match)["median"], 4)}
                if cv2 is not None:
                    ms = []
                    for _ in range(max(3, args.steps // 4)):
                        t0 = time.perf_counter()
                        for b in range(B):
                            if name == "homography":
                                cv2.findHomography(a0[b], a1[b], cv2.RANSAC, THRESHOLD, maxIters=ITERATIONS)
                            else:
                                cv2.findFundamentalMat(a0[b], a1[b], cv2.FM_RANSAC, THRESHOLD, 0.999, ITERATIONS)
                        ms.append(1e3 * (time.perf_counter() - t0))
                    row["opencv_ms"] = stats(ms)
                else:
                    row["opencv_ms"] = "absent (cv2 not importable)"
                row.update(info)
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
