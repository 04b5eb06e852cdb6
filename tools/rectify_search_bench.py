"""Rectification search (DESIGN.md §20): data["rectify1_candidates"] against what a caller writes without it, alternating
in one process.

Workload: 8 pairs at 640x480 (indoor_ds, thr 0), weights from torch.manual_seed(0), uniform-random images as in
bench.py, and K = 4 candidates per pair: the quarter turns of `rotation_candidates`.
  search      `matcher(batch)` with rectify1_candidates [8, 4, 3, 3]: image0's backbone once, only each pair's winning
              candidate refined;
  flattened   `matcher(batch)` on the 32 candidate pairs with rectify1, then the host pick: per-candidate match counts
              read back, the best candidate of each pair chosen and its matches kept;
  plain       `matcher(batch)` on the 8 pairs, for reference.
Each arm: step ms (CUDA events, L2 written before every call; min / median / max), matches kept and peak device memory
above the inputs.  The `match_search` kernel ms per call comes from a timing pass of its own.  Prints one JSON line with
the GPU name and power limit.

    python tools/rectify_search_bench.py [--steps 20] [--warmup 3]
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

BATCH, H, W, K = 8, 480, 640, 4


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
    dev = require_gpu("rectify_search_bench")
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().to(dev)
    g = torch.Generator().manual_seed(1000)
    img0 = torch.rand(BATCH, 1, H, W, generator=g).to(dev)
    img1 = torch.rand(BATCH, 1, H, W, generator=g).to(dev)
    size = torch.tensor([[W, H]] * BATCH, dtype=torch.int32, device=dev)
    cands = loftr_b200.rotation_candidates(size, size)

    def search():
        d = {"image0": img0, "image1": img1, "rectify1_candidates": cands}
        model(d)
        return d

    def flattened():
        d = {"image0": img0.repeat_interleave(K, 0), "image1": img1.repeat_interleave(K, 0),
             "rectify1": cands.reshape(BATCH * K, 3, 3)}
        model(d)
        counts = torch.bincount(d["b_ids"], minlength=BATCH * K).view(BATCH, K).cpu()   # the host pick
        choice = counts.argmax(1).to(dev)
        keep = (d["b_ids"] % K) == choice[d["b_ids"] // K]
        return {k: d[k][keep] for k in ("b_ids", "i_ids", "j_ids", "mconf", "mkpts0_f", "mkpts1_f", "minside1")}

    def plain():
        d = {"image0": img0, "image1": img1}
        model(d)
        return d

    arms = {"search": search, "flattened": flattened, "plain": plain}
    ms, last = alternate(arms, args.steps, args.warmup)
    res = {name: {"step_ms": stats(ms[name]), "matches": int(last[name]["b_ids"].numel()),
                  "peak_MB": peak_mb(fn)} for name, fn in arms.items()}
    res["search"]["choice"] = last["search"]["rectify1_choice"].tolist()
    res["search"]["counts"] = last["search"]["rectify1_counts"].tolist()
    tags = tag_ms(search, runs=args.steps, flush=True)
    kern_ms = tags["match_search"][0] / tags["match_search"][1]
    out = {"tool": "rectify_search_bench", "steps": args.steps, **gpu_label(), "batch": BATCH, "hw": [H, W], "K": K,
           "l2": "256 MiB buffer written before every timed call", "arms": res,
           "match_search_kernel_ms": round(kern_ms, 4)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
