"""Point tracking along a frame chain (DESIGN.md §21): `match_points` on the stacked pairs against `extract_features` +
`match_points_features` on a bank of the frames, with and without a guide, alternating in one process.

Workload: a chain of 9 frames at 640x480 (indoor_ds, thr 0), i.e. the 8 consecutive pairs (t, t + 1), with Q = 1024
uniform-random sub-pixel points per pair.  Weights from torch.manual_seed(0) and uniform-random frames as in bench.py.
Arms:
  stacked        match_points on image0 = frames[0:8], image1 = frames[1:9] (the backbone runs on 16 images);
  bank           extract_features on the 9 frames + match_points_features over the pair list (9 backbone images);
  bank_guided    the same with an identity-homography guide of radius 32 pixels (a local search, as for video).
Per arm:
  step_ms        eager call, CUDA events, a 256 MiB buffer written before every step (min / median / max);
  tags_ms        per step, from a profiled pass of its own: match_query, score_lse, score_argmax and fine_merge;
  peak_gb        torch.cuda.max_memory_allocated of one step.
`bank_equals_stacked` says whether the bank arm's outputs equal the stacked arm's bit for bit.  Prints one JSON line
with the GPU name and power limit.

    python tools/track_bench.py [--steps 10] [--warmup 2]
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

FRAMES, H, W, Q, RADIUS = 9, 480, 640, 1024, 32.0
TAGS = ("match_query", "score_lse", "score_argmax", "fine_merge")
Q_KEYS = ("qpts0_f", "qpts1_c", "qpts1_f", "qexpec_f", "qconf", "q_i_ids", "q_j_ids", "qmutual", "qvalid", "qinside")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = require_gpu("track_bench")
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().to(dev)
    g = torch.Generator().manual_seed(1000)
    frames = torch.rand(FRAMES, 1, H, W, generator=g).to(dev)
    pairs = FRAMES - 1
    pts = (torch.rand(pairs, Q, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])).to(dev)
    idx0 = torch.arange(pairs, device=dev)
    idx1 = idx0 + 1
    guide = {"kind": "homography", "model": torch.eye(3, device=dev).repeat(pairs, 1, 1), "radius": RADIUS}

    def stacked():
        d = {"image0": frames[:pairs], "image1": frames[1:]}
        model.match_points(d, pts)
        return d

    def bank(gd=None):
        feats = model.extract_features(frames)
        return model.match_points_features(feats, idx0, feats, idx1, pts, guide=gd)

    arms = {"stacked": stacked, "bank": bank, "bank_guided": lambda: bank(guide)}
    step_ms, last = alternate(arms, args.steps, args.warmup)
    res = {}
    for name, fn in arms.items():
        tags = tag_ms(fn, runs=3, flush=True)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        d = last[name]
        res[name] = {"step_ms": stats(step_ms[name]),
                     "tags_ms": {t: round(tags.get(t, (0.0, 0))[0] / 3, 4) for t in TAGS},
                     "peak_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 3),
                     "answered": int(d["qinside"].sum()), "qvalid": int(d["qvalid"].sum())}
    same = all(torch.equal(torch.nan_to_num(last["bank"][k].float()), torch.nan_to_num(last["stacked"][k].float()))
               for k in Q_KEYS)
    print(json.dumps({"tool": "track_bench", "frames": FRAMES, "pairs": pairs, "hw": [H, W], "queries_per_pair": Q,
                      "config": "indoor_ds thr 0", "guide": f"identity homography, radius {RADIUS:g}",
                      "steps": args.steps, **gpu_label(), "l2": "256 MiB buffer written before every timed step",
                      "bank_equals_stacked": same, "arms": res}))


if __name__ == "__main__":
    main()
