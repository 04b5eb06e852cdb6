"""Split-precision backbone (`backbone_impl="b200"`) against the single-pass fp16 one (`"b200_fp16"`), alternating in
one process on the same seeded weights (indoor_ds, thr 0) and images:
  extract:   `extract_features` on 16 images of 640x480;
  matcher:   one `matcher(batch)` step at 8 pairs of 640x480;
  pair list: the 120 pairs of the 16 images through the bank (one extract_features, 15 match_features of 8 pairs),
             as in tools/pair_list_bench.py.
A 256 MiB buffer is written before every timed call (untimed; flushes the 50 MB L2); calls are timed with CUDA events
and reported as min / median / max over --reps.  Then, in a pass of its own, every backbone launch of a 16-image
forward of each mode under the profiler (tools/conv_bench.py's launch_us: median us over 5 forwards) with its
algorithmic TFLOP/s (2 * pixels * Cout * Cin * k^2; in fp16 mode each product is one MMA, so issued = algorithmic), and
the workspace bytes of each mode.  Prints a Markdown layer table and one JSON line with the GPU name and power limit.

    python tools/backbone_fp16_bench.py [--reps 5] [--warmup 1]
"""
import argparse
import ctypes as C
import itertools
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import loftr_b200  # noqa: E402
from conv_bench import LAYERS, launch_us  # noqa: E402
from loftr_b200 import _lib  # noqa: E402
from measure import gpu_label, require_gpu, stats, timed  # noqa: E402

N_IMAGES, H, W, BATCH = 16, 480, 640, 8
MODES = ("b200", "b200_fp16")


def layer_gflop(n, h, w):
    """Algorithmic GFLOP of the stem and of every convolution after it, in launch order."""
    out = [2 * n * (h // 2) * (w // 2) * 128 * 49 / 1e9]
    for _, cin, cout, k, s, div in LAYERS:
        ho, wo = (h // div + 2 * (k // 2) - k) // s + 1, (w // div + 2 * (k // 2) - k) // s + 1
        out.append(2 * n * ho * wo * cout * cin * k * k / 1e9)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    dev = require_gpu("backbone_fp16_bench")
    torch.manual_seed(0)
    cfg = loftr_b200.get_cfg("indoor_ds", thr=0.0)
    models = {"b200": loftr_b200.LoFTR(cfg, backbone_impl="b200").eval()}
    models["b200_fp16"] = loftr_b200.LoFTR(cfg, backbone_impl="b200_fp16").eval()
    models["b200_fp16"].load_state_dict(models["b200"].state_dict())
    models = {k: m.to(dev) for k, m in models.items()}
    g = torch.Generator().manual_seed(1000)
    images = torch.rand(N_IMAGES, 1, H, W, generator=g).to(dev)
    pairs = torch.tensor(list(itertools.combinations(range(N_IMAGES), 2)), device=dev)
    batches = [(pairs[s:s + BATCH, 0].contiguous(), pairs[s:s + BATCH, 1].contiguous())
               for s in range(0, len(pairs), BATCH)]
    step = {"image0": images[:BATCH], "image1": images[BATCH:]}

    def one_rep(model):
        bank, t_ext = timed(lambda: model.extract_features(images))
        d = dict(step)
        _, t_step = timed(lambda: model(d))
        t_list = t_ext
        for i0, i1 in batches:
            t_list += timed(lambda: model.match_features(bank, i0, bank, i1))[1]
        return t_ext, t_step, t_list, int(d["b_ids"].shape[0])

    for _ in range(args.warmup):
        for mode in MODES:
            one_rep(models[mode])
    res = {mode: {"extract16_ms": [], "matcher_b8_ms": [], "pair_list_ms": []} for mode in MODES}
    matches = {}
    for _ in range(args.reps):   # alternate: both modes see the same clocks and neighbours
        for mode in MODES:
            t_ext, t_step, t_list, m = one_rep(models[mode])
            res[mode]["extract16_ms"].append(t_ext)
            res[mode]["matcher_b8_ms"].append(t_step)
            res[mode]["pair_list_ms"].append(t_list)
            matches[mode] = m

    gflop = layer_gflop(N_IMAGES, H, W)
    names = ["stem 7x7 s2"] + [name for name, *_ in LAYERS]
    us, ws_bytes = {}, {}
    for mode in MODES:
        tc = models[mode]._tc_backbone
        us[mode], _ = launch_us(tc, images)
        w, _ = tc._pack()
        lib = _lib.load()
        fn = lib.lb_backbone_workspace_bytes_fp16 if mode == "b200_fp16" else lib.lb_backbone_workspace_bytes
        ws_bytes[mode] = int(fn(C.byref(w), N_IMAGES, H, W))

    info = gpu_label()
    print(f"# {info['gpu']} at {info['power_limit']}, {N_IMAGES} images {H}x{W}, median of 5 profiled forwards")
    print("| layer | GFLOP | split us | split TFLOP/s | fp16 us | fp16 TFLOP/s | speed-up |")
    print("|---|---|---|---|---|---|---|")
    for name, gf, a, b in zip(names, gflop, us["b200"], us["b200_fp16"]):
        print(f"| {name} | {gf:.1f} | {a:.0f} | {gf / a * 1e3:.0f} | {b:.0f} | {gf / b * 1e3:.0f} | {a / b:.2f} |")
    ta, tb = sum(us["b200"]), sum(us["b200_fp16"])
    print(f"| **all launches** | {sum(gflop):.0f} | **{ta:.0f}** | {sum(gflop) / ta * 1e3:.0f} | **{tb:.0f}** | "
          f"{sum(gflop) / tb * 1e3:.0f} | {ta / tb:.2f} |")
    out = {"tool": "backbone_fp16_bench", **info, "images": N_IMAGES, "hw": [H, W], "batch": BATCH, "reps": args.reps,
           "l2": "256 MiB buffer written before every timed call", "workspace_bytes_16x480x640": ws_bytes,
           "matches_b8": matches, "backbone_launch_us_total": {m: round(sum(us[m]), 1) for m in MODES}}
    for mode in MODES:
        out[mode] = {k: stats(v) for k, v in res[mode].items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
