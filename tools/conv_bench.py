#!/usr/bin/env python
"""Per-launch times of the backbone of one bench.py step (8 pairs = 16 images of 640x480 through lb_backbone_forward),
taken with torch.profiler (CUDA activities) in a run of their own after warm-up:
    python tools/conv_bench.py [--batch 8] [--h 480] [--w 640] [--reps 5]
One row per launch in execution order: the output-channel tile N the launch ran with (read from the kernel's name),
median us over --reps profiled forwards, issued GFLOP (3 products x k-steps x N tile, from shapes), issued TFLOP/s,
and the L2 -> shared-memory operand bytes of one launch, computed from shapes, for
the per-tap patch loads of gemm_split_kernel ("tap") and the once-per-channel-block halo of conv3x3_halo_kernel
("halo"; weights still per tap).  The halo column is filled for the stride-1 3x3 layers only."""
import argparse
import os
import re
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import loftr_b200  # noqa: E402
from loftr_b200.loftr import TensorCoreBackbone  # noqa: E402
from measure import gpu_label, require_gpu  # noqa: E402

# (name, Cin, Cout, ksize, stride, input-grid divisor) in lb_backbone_forward's launch order after the stem
LAYERS = [
    ("layer1.0.conv1", 128, 128, 3, 1, 2), ("layer1.0.conv2 +skip", 128, 128, 3, 1, 2),
    ("layer1.1.conv1", 128, 128, 3, 1, 2), ("layer1.1.conv2 +skip", 128, 128, 3, 1, 2),
    ("layer2.0.conv1 s2", 128, 196, 3, 2, 2), ("layer2.0.downsample 1x1 s2", 128, 196, 1, 2, 2),
    ("layer2.0.conv2 +skip", 196, 196, 3, 1, 4), ("layer2.1.conv1", 196, 196, 3, 1, 4),
    ("layer2.1.conv2 +skip", 196, 196, 3, 1, 4), ("layer3.0.conv1 s2", 196, 256, 3, 2, 4),
    ("layer3.0.downsample 1x1 s2", 196, 256, 1, 2, 4), ("layer3.0.conv2 +skip", 256, 256, 3, 1, 8),
    ("layer3.1.conv1", 256, 256, 3, 1, 8), ("layer3.1.conv2 +skip", 256, 256, 3, 1, 8),
    ("layer3_outconv 1x1", 256, 256, 1, 1, 8), ("layer2_outconv 1x1 + upsample", 196, 256, 1, 1, 4),
    ("layer2_outconv2.0", 256, 256, 3, 1, 4), ("layer2_outconv2.3", 256, 196, 3, 1, 4),
    ("layer1_outconv 1x1 + upsample", 128, 196, 1, 1, 2), ("layer1_outconv2.0", 196, 196, 3, 1, 2),
    ("layer1_outconv2.3", 196, 128, 3, 1, 2)]


def layer_counts(cin, cout, k, s, div, n, h, w, bn):
    """(issued GFLOP, per-tap bytes, halo bytes or None) of one launch with output-channel tile bn."""
    cb, rem = (cin // 64, cin % 64) if cin > 64 and 0 < cin % 64 <= 16 else ((cin + 63) // 64, 0)
    hin, win = h // div, w // div
    ho, wo = (hin + 2 * (k // 2) - k) // s + 1, (win + 2 * (k // 2) - k) // s + 1
    tiles = n * -(-ho // 8) * -(-wo // 16)
    taps = k * k
    ksteps = taps * (4 * cb + (1 if rem else 0))
    gflop = tiles * ksteps * 3 * 2 * 128 * 16 * bn / 1e9
    b_bytes = taps * (cb * 64 + (16 if rem else 0)) * bn * 2 * 2               # hi + lo weight tiles per output tile
    tap_bytes = tiles * (taps * (cb * 64 + (16 if rem else 0)) * 128 * 2 * 2 + b_bytes)
    halo = None
    if k == 3 and s == 1:
        halo = tiles * ((cb * 8 + (2 if rem else 0)) * 180 * 16 * 2 + b_bytes)
    return gflop, tap_bytes, halo


def launch_us(tc, img, reps=5):
    """Median us of every backbone launch of `tc(img)` (stem first) over `reps` profiled forwards after 3 warm-up
    forwards, and the kernel names of those launches."""
    for _ in range(3):
        tc(img)
    torch.cuda.synchronize()
    per_rep = []
    for _ in range(reps):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            tc(img)
            torch.cuda.synchronize()
        ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and ("EpiConv" in e.name or "conv_stem" in e.name)), key=lambda e: e.time_range.start)
        per_rep.append([e.time_range.elapsed_us() for e in ev])
    if {len(r) for r in per_rep} != {len(LAYERS) + 1}:
        sys.exit(f"expected {len(LAYERS) + 1} backbone launches per forward, got {sorted({len(r) for r in per_rep})}")
    return [statistics.median(r[i] for r in per_rep) for i in range(len(LAYERS) + 1)], [e.name for e in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8, help="image pairs (2x as many images)")
    ap.add_argument("--h", type=int, default=480)
    ap.add_argument("--w", type=int, default=640)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    require_gpu("conv_bench")
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().cuda()
    tc = TensorCoreBackbone(model.backbone)
    n = 2 * args.batch
    img = torch.rand(n, 1, args.h, args.w, generator=torch.Generator().manual_seed(1000)).cuda()
    us, names = launch_us(tc, img, args.reps)
    # output-channel tile of each EpiConv launch: the BLOCK_N template argument in the (de)mangled kernel name
    tiles_n = [int(m.group(1)) for m in (re.search(r"EpiConv(?:<|ILi)(\d+)", name) for name in names) if m]
    if len(tiles_n) != len(LAYERS):
        sys.exit(f"expected {len(LAYERS)} launches named EpiConv<N> per forward, got {len(tiles_n)}")
    info = gpu_label()
    print(f"# {info['gpu']} at {info['power_limit']}, {n} images {args.h}x{args.w}, median of {args.reps} profiled "
          "forwards")
    print("| layer | N tile | us | issued GFLOP | issued TFLOP/s | L2->smem MB (tap) | L2->smem MB (halo) |")
    print("|---|---|---|---|---|---|---|")
    print(f"| stem 7x7 s2 | - | {us[0]:.0f} | - | - | - | - |")
    tot, tot_s1 = us[0], 0.0
    for (name, cin, cout, k, s, div), bn, t in zip(LAYERS, tiles_n, us[1:]):
        gf, tb, hb = layer_counts(cin, cout, k, s, div, n, args.h, args.w, bn)
        tot += t
        if hb is not None:
            tot_s1 += t
        print(f"| {name} | {bn} | {t:.0f} | {gf:.0f} | {gf / t * 1e3:.0f} | {tb / 1e6:.0f} | "
              f"{'-' if hb is None else f'{hb / 1e6:.0f}'} |")
    print(f"| **all launches** | | **{tot:.0f}** | | | | |")
    print(f"| **stride-1 3x3 only** | | **{tot_s1:.0f}** | | | | |")


if __name__ == "__main__":
    main()
