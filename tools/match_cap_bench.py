"""Per-pair match cap (`match_coarse.max_matches_per_pair`): step time, select-kernel time, matches and memory with
k = none, 256 and 1024, alternating in one process.

Workloads: 8 x 640x480 and 1 x 1280x960 (indoor_ds, thr 0), and 4 x 832x832 with a different padding mask per image
(outdoor_ds, thr 0), with weights from torch.manual_seed(0) and uniform-random images as in bench.py.  Per workload
and k:
  step_ms             eager `model(data)`, CUDA events, a 256 MiB buffer written before every step (min / median / max);
  match_cap_ms        the select kernel per step (`match_cap` timing tag), next to the score kernels of the coarse
                      matching (`score_lse` + `score_argmax`), from a profiled pass of its own;
  matches_per_pair    before (k = none) and after the cap (min / mean / max over the pairs);
  captured_capacity   the default capacity of `CapturedMatcher`, and the peak device memory
                      (torch.cuda.max_memory_allocated) of its construction and one replay, and of one eager step.
Prints one JSON line with the GPU name and power limit.

    python tools/match_cap_bench.py [--steps 10] [--warmup 2]
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

CAPS = [None, 256, 1024]
# (name, config, batch, H, W, valid (h, w) of image0 / image1 per pair or None)
WORKLOADS = [
    ("8x640x480", "indoor_ds", 8, 480, 640, None),
    ("1x1280x960", "indoor_ds", 1, 960, 1280, None),
    ("4x832x832_masked", "outdoor_ds", 4, 832, 832,
     ([(832, 624), (832, 832), (560, 832), (704, 768)], [(640, 832), (768, 832), (832, 832), (832, 616)])),
]


def inputs(batch, h, w, valid, dev):
    g = torch.Generator().manual_seed(1000)
    data = {"image0": torch.rand(batch, 1, h, w, generator=g), "image1": torch.rand(batch, 1, h, w, generator=g)}
    if valid is not None:   # MegaDepth-style padding: zeroed images outside the valid region, coarse bool masks
        for side, regions in enumerate(valid):
            mask = torch.zeros(batch, h // 8, w // 8, dtype=torch.bool)
            for b, (vh, vw) in enumerate(regions):
                mask[b, : vh // 8, : vw // 8] = True
                data[f"image{side}"][b, :, vh:, :] = 0
                data[f"image{side}"][b, :, :, vw:] = 0
            data[f"mask{side}"] = mask
    return {k: v.to(dev) for k, v in data.items()}


def run(name, cfg_name, batch, h, w, valid, steps, warmup, dev):
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg(cfg_name, thr=0.0)).eval().to(dev)
    inp = inputs(batch, h, w, valid, dev)
    cmatch = model.coarse_matching

    def step(k):
        cmatch.max_matches_per_pair = k
        d = dict(inp)
        model(d)
        return d

    step_ms, last = alternate({k: (lambda k=k: step(k)) for k in CAPS}, steps, warmup)

    kernel = {}
    for k in CAPS:
        tags = tag_ms(lambda: step(k), runs=3, flush=True)
        cap_ms, cap_n = tags.get("match_cap", (0.0, 0))
        score_ms = tags.get("score_lse", (0.0, 0))[0] + tags.get("score_argmax", (0.0, 0))[0]
        kernel[k] = {"match_cap_ms_per_step": round(cap_ms / 3, 4), "match_cap_launches_per_step": cap_n / 3,
                     "score_kernels_ms_per_step": round(score_ms / 3, 4)}

    memory = {}
    for k in CAPS:
        cmatch.max_matches_per_pair = k
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        step(k)
        torch.cuda.synchronize()
        eager_peak = torch.cuda.max_memory_allocated()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        cm = loftr_b200.CapturedMatcher(model, batch, (h, w), masks=valid is not None)
        cm(dict(inp))
        torch.cuda.synchronize()
        memory[k] = {"captured_capacity": cm.capacity,
                     "captured_peak_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 3),
                     "eager_peak_gb": round(eager_peak / 2 ** 30, 3)}
        del cm
        torch.cuda.empty_cache()

    def per_pair(d):
        c = torch.bincount(d["b_ids"], minlength=batch).float()
        return {"min": int(c.min()), "mean": round(float(c.mean()), 1), "max": int(c.max())}

    res = {"workload": name, "config": cfg_name, "batch": batch, "hw": [h, w], "masked": valid is not None,
           "L": (h // 8) * (w // 8), "caps": {}}
    for k in CAPS:
        res["caps"]["none" if k is None else str(k)] = {"step_ms": stats(step_ms[k]),
                                                         "matches_per_pair": per_pair(last[k]), **kernel[k],
                                                         **memory[k]}
    del model, last
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = require_gpu("match_cap_bench")
    out = {"tool": "match_cap_bench", "steps": args.steps, **gpu_label(),
           "l2": "256 MiB buffer written before every timed step",
           "workloads": [run(*w, args.steps, args.warmup, dev) for w in WORKLOADS]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
