"""Eager `model(data)` against `loftr_b200.CapturedMatcher` (one CUDA-graph replay per step), alternating in one
process.  Per workload: GPU ms per step (CUDA events), host wall ms per step (ending in a device synchronise), library
kernel launches per step (enqueued by the host; a graph replay enqueues none) and whether both produced bit-identical
outputs.  indoor_ds at thr 0 with seeded weights and uniform-random images, as in bench.py.  Prints one JSON line with
the GPU name and power limit (read-only nvidia-smi query).

    python tools/graph_bench.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import loftr_b200  # noqa: E402
from loftr_b200 import _lib  # noqa: E402

WORKLOADS = [(1, 240, 320), (1, 480, 640), (1, 960, 1280), (8, 480, 640)]   # (batch, H, W)
KEYS = ["b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f", "expec_f", "gt_mask"]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], check=True,
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the numbers stay valid; say where the label is missing
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({type(e).__name__})"}


def run(batch, h, w, steps, warmup, dev):
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().to(dev)
    g = torch.Generator().manual_seed(1000)
    img0 = torch.rand(batch, 1, h, w, generator=g).to(dev)
    img1 = torch.rand(batch, 1, h, w, generator=g).to(dev)
    cm = loftr_b200.CapturedMatcher(model, batch, (h, w))
    lib = _lib.load()

    def eager():
        d = {"image0": img0, "image1": img1}
        model(d)
        return d

    def captured():
        d = {"image0": img0, "image1": img1}
        cm(d)
        return d

    stats = {}
    for name, fn in (("eager", eager), ("graph", captured)):
        for _ in range(warmup):
            fn()
        stats[name] = {"gpu_ms": [], "wall_ms": [], "launches": []}
    torch.cuda.synchronize()
    last = {}
    for _ in range(steps):
        for name, fn in (("eager", eager), ("graph", captured)):   # alternate: both see the same clocks
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n0 = lib.lb_launch_count()
            t0 = time.perf_counter()
            e0.record()
            last[name] = fn()
            e1.record()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            stats[name]["gpu_ms"].append(e0.elapsed_time(e1))
            stats[name]["wall_ms"].append((t1 - t0) * 1e3)
            stats[name]["launches"].append(lib.lb_launch_count() - n0)
    equal = all(torch.equal(last["eager"][k], last["graph"][k]) for k in KEYS)
    med = lambda v: sorted(v)[len(v) // 2]
    res = {"batch": batch, "hw": [h, w], "matches": int(last["eager"]["b_ids"].shape[0]),
           "capacity": cm.capacity, "outputs_equal": equal}
    for name, s in stats.items():
        res[name] = {"gpu_ms_median": round(med(s["gpu_ms"]), 3), "wall_ms_median": round(med(s["wall_ms"]), 3),
                     "lib_launches_per_step": med(s["launches"])}
    res["wall_speedup"] = round(res["eager"]["wall_ms_median"] / res["graph"]["wall_ms_median"], 3)
    del cm, model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("graph_bench: no CUDA device (this measurement needs an H100)")
    dev = torch.device("cuda:0")
    out = {"tool": "graph_bench", "steps": args.steps, **gpu_info(),
           "workloads": [run(b, h, w, args.steps, args.warmup, dev) for b, h, w in WORKLOADS]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
