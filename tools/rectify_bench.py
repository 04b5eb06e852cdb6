"""Rectified matching (DESIGN.md §19): the cost of data["rectify1"], alternating with the plain call in one process.

Workload: 8 pairs at 640x480 (indoor_ds, thr 0), weights from torch.manual_seed(0), uniform-random images as in
bench.py, and per pair a homography about the image centres (rotation 10 deg, zoom 1.1, a small perspective row).
  warp   lb_rectify_images alone (`warp_images`): call ms (CUDA events, L2 written before every call; min / median /
         max), `rectify` kernel ms from a timing pass of its own, and the bytes the warp must move: the output written
         once plus image1 read once (the bilinear taps of neighbouring pixels overlap, so each input pixel needs one
         read from DRAM), over the kernel time;
  step   `matcher(batch)` with and without rectify1: step ms (min / median / max), matches, and the extra device
         memory of the rectified call (peak, one image buffer expected).
Prints one JSON line with the GPU name and power limit.

    python tools/rectify_bench.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import loftr_b200  # noqa: E402
from measure import alternate, gpu_label, require_gpu, stats, tag_ms  # noqa: E402

BATCH, H, W = 8, 480, 640


def models(dev):
    a, z = math.radians(10.0), 1.1
    c = ((W - 1) / 2, (H - 1) / 2)
    t0 = torch.tensor([[1, 0, -c[0]], [0, 1, -c[1]], [0, 0, 1]], dtype=torch.float64)
    t1 = torch.tensor([[1, 0, c[0]], [0, 1, c[1]], [0, 0, 1]], dtype=torch.float64)
    r = torch.tensor([[z * math.cos(a), -z * math.sin(a), 0], [z * math.sin(a), z * math.cos(a), 0], [1e-4, -5e-5, 1]],
                     dtype=torch.float64)
    return (t1 @ r @ t0).float().to(dev).repeat(BATCH, 1, 1)


def peak_mb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = require_gpu("rectify_bench")
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().to(dev)
    g = torch.Generator().manual_seed(1000)
    img0 = torch.rand(BATCH, 1, H, W, generator=g).to(dev)
    img1 = torch.rand(BATCH, 1, H, W, generator=g).to(dev)
    rect = models(dev)

    warp = {"warp": lambda: loftr_b200.warp_images(img1, rect, (H, W))}
    ms, _ = alternate(warp, args.steps, args.warmup)
    tags = tag_ms(warp["warp"], runs=args.steps, flush=True)
    kern_ms = tags["rectify"][0] / tags["rectify"][1]
    nbytes = 2 * BATCH * H * W * 4   # output written once, image1 read once
    warp_res = {"call_ms": stats(ms["warp"]), "rectify_kernel_ms": round(kern_ms, 4), "bytes": nbytes,
                "achieved_GBps": round(nbytes / (kern_ms * 1e-3) / 1e9, 1)}

    def step(rectified):
        d = {"image0": img0, "image1": img1}
        if rectified:
            d["rectify1"] = rect
        model(d)
        return d
    arms = {"plain": lambda: step(False), "rectified": lambda: step(True)}
    ms, last = alternate(arms, args.steps, args.warmup)
    step_res = {name: {"step_ms": stats(ms[name]), "matches": int(last[name]["b_ids"].numel()),
                       "peak_extra_MB": peak_mb(fn)} for name, fn in arms.items()}
    step_res["rectified"]["inside"] = int(last["rectified"]["minside1"].sum())
    out = {"tool": "rectify_bench", "steps": args.steps, **gpu_label(), "batch": BATCH, "hw": [H, W],
           "l2": "256 MiB buffer written before every timed call", "warp": warp_res, "step": step_res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
