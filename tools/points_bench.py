"""`LoFTR.match_points` (DESIGN.md §17) next to the forward: step time, tagged kernel time and peak memory at
8 x 640x480 (indoor_ds, thr 0) for Q = 256, 1024 and 4800 queries per pair, alternating with `matcher(batch)` in one
process.

Weights from torch.manual_seed(0) and uniform-random images as in bench.py; the queries are uniform-random sub-pixel
points over image0 (every one inside).  Per arm:
  step_ms        eager call, CUDA events, a 256 MiB buffer written before every step (min / median / max);
  tags_ms        per step, from a profiled pass of its own: match_query (the point-to-cell kernel), score_lse +
                 score_argmax (the coarse score passes) and fine_merge (the fine windows' merge product);
  peak_gb        torch.cuda.max_memory_allocated of one step.
Prints one JSON line with the GPU name and power limit.

    python tools/points_bench.py [--steps 10] [--warmup 2]
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

BATCH, H, W = 8, 480, 640
QUERIES = [256, 1024, 4800]
TAGS = ("match_query", "score_lse", "score_argmax", "fine_merge")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = require_gpu("points_bench")
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().to(dev)
    g = torch.Generator().manual_seed(1000)
    inp = {"image0": torch.rand(BATCH, 1, H, W, generator=g).to(dev),
           "image1": torch.rand(BATCH, 1, H, W, generator=g).to(dev)}
    pts = {q: (torch.rand(BATCH, q, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])).to(dev) for q in QUERIES}

    def forward():
        d = dict(inp)
        model(d)
        return d

    def points(q):
        d = dict(inp)
        model.match_points(d, pts[q])
        return d

    arms = {"forward": forward, **{f"match_points_q{q}": (lambda q=q: points(q)) for q in QUERIES}}
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
    res["forward"]["matches"] = int(last["forward"]["b_ids"].shape[0])
    for q in QUERIES:
        d = last[f"match_points_q{q}"]
        res[f"match_points_q{q}"].update({"queries": BATCH * q, "answered": int(d["qinside"].sum()),
                                          "qvalid": int(d["qvalid"].sum())})
    print(json.dumps({"tool": "points_bench", "batch": BATCH, "hw": [H, W], "config": "indoor_ds thr 0",
                      "steps": args.steps, **gpu_label(), "l2": "256 MiB buffer written before every timed step",
                      "arms": res}))


if __name__ == "__main__":
    main()
