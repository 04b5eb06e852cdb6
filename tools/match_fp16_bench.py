"""Split-precision matching (`match_precision="split"`) against the single-pass fp16 mode (`"fp16"`), alternating in
one process on the same seeded weights and images.  Workloads (`matcher(batch)` steps, thr 0):
  grid:     the four backbone_impl x match_precision combinations at 8 pairs of 640x480, indoor_ds (linear attention,
            dual-softmax);
  ot:       split / fp16 matching (b200 backbone) at 8 x 640x480, indoor_ot (Sinkhorn);
  full:     split / fp16 matching (b200 backbone) at 8 x 640x480, indoor_ds with full attention in both transformers;
  n1_1280:  split / fp16 matching (b200 backbone) at 1 pair of 1280x960, indoor_ds.
A 256 MiB buffer is written before every timed call (untimed; flushes the 50 MB L2); steps are timed with CUDA events
after --warmup untimed rounds and reported as min / median / max over --reps.  Then, in a pass of its own, the
per-tag kernel ms of one step of each workload and mode (lb_timing_*, CUDA events around every tagged launch).  Prints
one JSON line with the GPU name and power limit.

    python tools/match_fp16_bench.py [--reps 7] [--warmup 2]
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

TAGS = ("proj_act", "tf_kv_proj_fused", "tf_q_attn_fused", "merge_ln", "mlp1_relu", "mlp2_ln_res", "tf_full_attn",
        "score_lse", "score_argmax")


def workloads():
    """name -> (config, batch, (H, W), [(backbone_impl, match_precision), ...])"""
    ds = loftr_b200.get_cfg("indoor_ds", thr=0.0)
    full = loftr_b200.get_cfg("indoor_ds", thr=0.0)
    full["coarse"]["attention"] = full["fine"]["attention"] = "full"
    both = [("b200", "split"), ("b200", "fp16")]
    return {"grid": (ds, 8, (480, 640), [(b, p) for b in ("b200", "b200_fp16") for p in ("split", "fp16")]),
            "ot": (loftr_b200.get_cfg("indoor_ot", thr=0.0), 8, (480, 640), both),
            "full": (full, 8, (480, 640), both),
            "n1_1280": (ds, 1, (960, 1280), both)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    args = ap.parse_args()
    dev = require_gpu("match_fp16_bench")
    out = {"tool": "match_fp16_bench", **gpu_label(), "reps": args.reps, "warmup": args.warmup,
           "l2": "256 MiB buffer written before every timed call"}
    for name, (cfg, n, (h, w), modes) in workloads().items():
        if args.only and name not in args.only.split(","):
            continue
        torch.manual_seed(0)
        ref = loftr_b200.LoFTR(cfg, backbone_impl="b200").eval()
        models = {}
        for b, p in modes:
            m = loftr_b200.LoFTR(cfg, backbone_impl=b, match_precision=p).eval()
            m.load_state_dict(ref.state_dict())
            models[f"{b}/{p}"] = m.to(dev)
        g = torch.Generator().manual_seed(1000)
        step = {"image0": torch.rand(n, 1, h, w, generator=g).to(dev),
                "image1": torch.rand(n, 1, h, w, generator=g).to(dev)}

        def run(model):
            d = dict(step)
            model(d)
            return d

        arms = {k: (lambda m=m: run(m)) for k, m in models.items()}
        times, last = alternate(arms, args.reps, args.warmup)
        matches = {k: int(d["b_ids"].shape[0]) for k, d in last.items()}
        tags = {}
        for k, fn in arms.items():
            rec = tag_ms(fn, flush=True)
            tags[k] = {t: round(rec[t][0], 3) for t in TAGS if rec.get(t, (0, 0))[1]}
        out[name] = {"batch": n, "hw": [h, w], "match_type": cfg["match_coarse"]["match_type"],
                     "attention": cfg["coarse"]["attention"], "step_ms": {k: stats(v) for k, v in times.items()},
                     "matches": matches, "tag_ms": tags}
        print(json.dumps({name: out[name]}), flush=True)
        del models
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
