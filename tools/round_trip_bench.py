"""Forward-backward track checks along a frame chain (DESIGN.md §22): `match_points_features` alone, with
`round_trip=True`, and the two-call check on the swapped pairs, alternating in one process.

Workload: the chain of tools/track_bench.py: 9 frames at 640x480 (indoor_ds, thr 0), the 8 consecutive pairs
(t, t + 1), Q = 1024 uniform-random sub-pixel points per pair; weights from torch.manual_seed(0), uniform-random
frames.  Every arm runs `extract_features` on the 9 frames first, as a tracker does per step.
Arms:
  forward      match_points_features over the pair list (one leg);
  round_trip   the same with round_trip=True: the answers are queried back from image1 on the same coarse pass;
  swapped      the forward, then match_points_features on the swapped pairs (t + 1, t) at qpts1_f with valid0 =
               qinside: the check as a second full match.
Per arm:
  step_ms      eager call, CUDA events, a 256 MiB buffer written before every step (min / median / max);
  tags_ms      per step, from a profiled pass of its own: match_query, score_lse, score_argmax and fine_merge;
  peak_gb      torch.cuda.max_memory_allocated of one step.
`back_leg_equals_image1_call` says whether the round-trip arm's back leg equals a separate image1-side call at its
first answers (points1 = qpts1_f, valid1 = qinside) bit for bit.  Prints one JSON line with the GPU name and power
limit.

    python tools/round_trip_bench.py [--steps 10] [--warmup 2]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import loftr_b200  # noqa: E402
from measure import alternate, gpu_label, require_gpu, stats, tag_ms  # noqa: E402

FRAMES, H, W, Q = 9, 480, 640, 1024
TAGS = ("match_query", "score_lse", "score_argmax", "fine_merge")


def _same(a, b):
    a, b = a.float(), b.float()
    return torch.equal(torch.nan_to_num(a), torch.nan_to_num(b)) and torch.equal(torch.isnan(a), torch.isnan(b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = require_gpu("round_trip_bench")
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().to(dev)
    g = torch.Generator().manual_seed(1000)
    frames = torch.rand(FRAMES, 1, H, W, generator=g).to(dev)
    pairs = FRAMES - 1
    pts = (torch.rand(pairs, Q, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])).to(dev)
    idx0 = torch.arange(pairs, device=dev)
    idx1 = idx0 + 1

    def forward(round_trip=False):
        feats = model.extract_features(frames)
        return model.match_points_features(feats, idx0, feats, idx1, pts, round_trip=round_trip)

    def swapped():
        feats = model.extract_features(frames)
        out = model.match_points_features(feats, idx0, feats, idx1, pts)
        return model.match_points_features(feats, idx1, feats, idx0, out["qpts1_f"], out["qinside"])

    arms = {"forward": forward, "round_trip": lambda: forward(True), "swapped": swapped}
    step_ms, last = alternate(arms, args.steps, args.warmup)
    res = {}
    for name, fn in arms.items():
        tags = tag_ms(fn, runs=3, flush=True)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        res[name] = {"step_ms": stats(step_ms[name]),
                     "tags_ms": {t: round(tags.get(t, (0.0, 0))[0] / 3, 4) for t in TAGS},
                     "peak_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)}
    rt = last["round_trip"]
    feats = model.extract_features(frames)
    sep = model.match_points_features(feats, idx0, feats, idx1, points1=rt["qpts1_f"], valid1=rt["qinside"])
    same = all(_same(rt[k], sep[r]) for k, r in (("qback_pts", "qpts0_f"), ("qback_conf", "qconf"),
                                                  ("qback_valid", "qvalid"), ("qback_inside", "qinside")))
    back = rt["qback_inside"]
    print(json.dumps({"tool": "round_trip_bench", "frames": FRAMES, "pairs": pairs, "hw": [H, W],
                      "queries_per_pair": Q, "config": "indoor_ds thr 0", "steps": args.steps, **gpu_label(),
                      "l2": "256 MiB buffer written before every timed step",
                      "back_leg_equals_image1_call": same, "answered": int(rt["qinside"].sum()),
                      "back_answered": int(back.sum()),
                      "median_fb_err_px": round(rt["qfb_err"][back].median().item(), 3) if back.any() else None,
                      "arms": res}))


if __name__ == "__main__":
    main()
