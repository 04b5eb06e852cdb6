"""Guided coarse matching (DESIGN.md §18): the cost of the guide in the score epilogues, unguided against guided,
alternating in one process.

Workload: 8 pairs at 640x480 (indoor_ds and indoor_ot, thr 0), weights from torch.manual_seed(0), uniform-random
images as in bench.py.
  coarse      CoarseMatching.run on the coarse transformer's output planes: lb_coarse_match (or
              lb_coarse_match_fp16) against lb_coarse_match_guided, for dual-softmax and Sinkhorn, split and fp16, with
              a homography guide (identity, radius 64 px: a motion prior of 8 cells); call_ms (CUDA events, L2 written
              before every call; min / median / max) and the score kernels' time per call (`score_lse` + `score_argmax`
              timing tags, from a pass of its own);
  step        a whole `match_features` call on a bank of the 16 images, unguided against guided by the fundamental
              matrix its own `estimate="fundamental"` call returned (radius 16 px): the two-pass use of DESIGN.md §18.
Every score tile is still computed: no speed-up is expected, only the predicate's ALU work in the epilogues.
Prints one JSON line with the GPU name and power limit.

    python tools/guided_bench.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import loftr_b200  # noqa: E402
from loftr_b200.loftr import CoarseMatching, split_planes  # noqa: E402
from measure import alternate, gpu_label, require_gpu, stats, tag_ms  # noqa: E402

BATCH, H, W = 8, 480, 640


def coarse_arms(cfg_name, steps, warmup, dev):
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg(cfg_name, thr=0.0)).eval().to(dev)
    model.expose_coarse_features = True
    g = torch.Generator().manual_seed(1000)
    data = {"image0": torch.rand(BATCH, 1, H, W, generator=g).to(dev),
            "image1": torch.rand(BATCH, 1, H, W, generator=g).to(dev)}
    model(data)
    f0, f1 = data["_feat_c0"], data["_feat_c1"]
    n, L, c = f0.shape
    S = f1.shape[1]
    hi, lo = split_planes(torch.cat([f0.reshape(n * L, c), f1.reshape(n * S, c)]).contiguous())
    base = {k: data[k] for k in ("hw0_i", "hw1_i", "hw0_c", "hw1_c")}
    guide = {"kind": "homography", "model": torch.eye(3, device=dev).repeat(n, 1, 1), "radius": 64.0}
    out = {}
    for precision in ("split", "fp16"):
        cm = CoarseMatching(model.config["match_coarse"], precision=precision).eval().to(dev)
        cm.load_state_dict(model.coarse_matching.state_dict())

        def call(gd):
            d = dict(base)
            if gd is not None:
                d["guide"] = gd
            cm.run(hi, lo, c, n, L, S, c, d)
            return d
        arms = {"unguided": lambda: call(None), "guided": lambda: call(guide)}
        ms, last = alternate(arms, steps, warmup)
        res = {}
        for name, fn in arms.items():
            tags = tag_ms(fn, runs=3, flush=True)
            score = tags.get("score_lse", (0.0, 0))[0] + tags.get("score_argmax", (0.0, 0))[0]
            res[name] = {"call_ms": stats(ms[name]), "score_kernels_ms": round(score / 3, 4),
                         "matches": int(last[name]["b_ids"].numel())}
        out[precision] = res
    return out


def step_arms(steps, warmup, dev):
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().to(dev)
    g = torch.Generator().manual_seed(1000)
    bank = model.extract_features(torch.rand(2 * BATCH, 1, H, W, generator=g).to(dev))
    i0 = torch.arange(BATCH, device=dev)
    i1 = i0 + BATCH
    first = model.match_features(bank, i0, bank, i1, estimate="fundamental")
    guide = {"kind": "fundamental", "model": first["geom_model"], "radius": 16.0}
    arms = {"unguided": lambda: model.match_features(bank, i0, bank, i1),
            "guided": lambda: model.match_features(bank, i0, bank, i1, guide=guide)}
    ms, last = alternate(arms, steps, warmup)
    return {name: {"step_ms": stats(ms[name]), "matches": int(last[name]["b_ids"].numel())} for name in arms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = require_gpu("guided_bench")
    out = {"tool": "guided_bench", "steps": args.steps, **gpu_label(), "batch": BATCH, "hw": [H, W],
           "l2": "256 MiB buffer written before every timed call",
           "coarse": {"dual_softmax": coarse_arms("indoor_ds", args.steps, args.warmup, dev),
                      "sinkhorn": coarse_arms("indoor_ot", args.steps, args.warmup, dev)},
           "match_features_step": step_arms(args.steps, args.warmup, dev)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
