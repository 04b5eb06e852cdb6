"""All-linear against all-full attention, alternating in one process on the same seeded model weights and inputs.
Per workload: step ms as min / median / max (CUDA events, L2 flushed before every step as in bench.py), the full-attention coarse kernel's
ms per launch (timing tag `tf_full_attn`) and its algorithmic rate, 4*L*S*C FLOP per query set and layer call, counted
once (the three split-precision MMAs are not counted: their ceiling is 1/3 of the fp16 dense peak).  indoor_ds at
thr 0 with uniform-random images.  Prints one JSON line per workload with the GPU name and power limit (read-only
nvidia-smi query).

    python tools/full_attention_bench.py [--steps 10] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import loftr_b200  # noqa: E402
from loftr_b200 import _lib  # noqa: E402

WORKLOADS = [(8, 480, 640), (1, 960, 1280)]   # (batch, H, W)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], check=True,
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({type(e).__name__})"}


def make_model(attention, dev, state=None):
    cfg = loftr_b200.get_cfg("indoor_ds", thr=0.0)
    cfg["coarse"]["attention"] = cfg["fine"]["attention"] = attention
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(cfg).eval()
    if state is not None:
        model.load_state_dict(state)
    return model.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    linear = make_model("linear", dev)
    full = make_model("full", dev, {k: v.cpu() for k, v in linear.state_dict().items()})
    models = {"linear": linear, "full": full}
    for batch, h, w in WORKLOADS:
        g = torch.Generator().manual_seed(1000)
        img0 = torch.rand(batch, 1, h, w, generator=g).to(dev)
        img1 = torch.rand(batch, 1, h, w, generator=g).to(dev)
        ms = {k: [] for k in models}
        matches = {}
        for name, m in models.items():
            for _ in range(args.warmup):
                m({"image0": img0, "image1": img1})
        for _ in range(args.steps):
            for name, m in models.items():   # alternating runs
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                d = {"image0": img0, "image1": img1}
                e0.record()
                m(d)
                e1.record()
                e1.synchronize()
                ms[name].append(e0.elapsed_time(e1))
                matches[name] = int(d["b_ids"].shape[0])
        # per-launch kernel time of the coarse full-attention kernel (separate, timed steps)
        _lib.timing_enable(True)
        for _ in range(2):
            full({"image0": img0, "image1": img1})
        torch.cuda.synchronize()
        t = _lib.timing_collect()
        _lib.timing_enable(False)
        k_ms, k_n = t["tf_full_attn"]
        L = (h // 8) * (w // 8)
        per_launch = k_ms / max(k_n, 1)
        # one launch = one layer call over n_groups query sets: self passes cover 2*batch sets, cross passes batch
        n_layers = len(full.loftr_coarse.layer_names)
        flop_per_step = 4.0 * L * L * 256 * 2 * batch * n_layers
        launches_per_step = k_n / 2
        spread = lambda v: [round(min(v), 2), round(sorted(v)[len(v) // 2], 2), round(max(v), 2)]
        print(json.dumps({
            "workload": f"{batch}x{w}x{h}", "L": L, **info,
            "step_ms_linear_min_med_max": spread(ms["linear"]), "step_ms_full_min_med_max": spread(ms["full"]),
            "matches_linear": matches["linear"], "matches_full": matches["full"],
            "full_attn_ms_per_launch": round(per_launch, 3), "full_attn_launches_per_step": launches_per_step,
            "full_attn_ms_per_step": round(k_ms / 2, 2),
            "full_attn_tflops": round(flop_per_step / (k_ms / 2 * 1e-3) / 1e12, 1),
            "gflop_per_image_per_layer_call": round(4.0 * L * L * 256 / 1e9, 2),
        }), flush=True)


if __name__ == "__main__":
    main()
