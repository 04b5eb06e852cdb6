#!/usr/bin/env python
"""Per-layer backbone table from an ncu launch list of one step (tools/profile_step.py, batch 8 x 640x480):
    python tools/conv_layer_table.py <launches>.csv [more.csv ...]
Launch ids 1..22 of a step are the stem and the 21 convolutions in execution order."""
import csv
import sys

LAYERS = [  # (name, issued GFLOP at batch 8: 3 products x k-steps x N tile, None for the stem)
    ("stem 7x7 s2 1->128", None), ("layer1.0.conv1", 1087), ("layer1.0.conv2 +skip", 1087), ("layer1.1.conv1", 1087),
    ("layer1.1.conv2 +skip", 1087), ("layer2.0.conv1 s2", 442), ("layer2.0.downsample 1x1 s2", 49),
    ("layer2.0.conv2 +skip", 718), ("layer2.1.conv1", 718), ("layer2.1.conv2 +skip", 718), ("layer3.0.conv1 s2", 221),
    ("layer3.0.downsample 1x1 s2", 25), ("layer3.0.conv2 +skip", 272), ("layer3.1.conv1", 272),
    ("layer3.1.conv2 +skip", 272), ("layer3_outconv 1x1", 30), ("layer2_outconv 1x1 + upsample", 98),
    ("layer2_outconv2.0", 1087), ("layer2_outconv2.3", 883), ("layer1_outconv 1x1 + upsample", 196),
    ("layer1_outconv2.0", 2871), ("layer1_outconv2.3", 1767)]
PEAK = 989.0  # H100 SXM data sheet, dense bf16 TFLOP/s (an upper bound, not reached)


def load(path):
    rows = list(csv.reader(open(path)))
    hdr = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    return [int(r[-1]) for r in rows[hdr + 1:] if len(r) > 14]


cols = [load(p) for p in sys.argv[1:]]
print("| layer | issued GFLOP | " + " | ".join(f"{p.split('/')[-1]} us (eff)" for p in sys.argv[1:]) + " |")
print("|---|---|" + "---|" * len(cols))
tot = [0] * len(cols)
for i, (name, gf) in enumerate(LAYERS):
    cells = []
    for c, t in enumerate(cols):
        us = t[1 + i] / 1e3
        tot[c] += us
        cells.append(f"{us:.0f}" + (f" ({gf / us * 1e3 / PEAK:.2f})" if gf else ""))
    print(f"| {name} | {gf if gf else '-'} | " + " | ".join(cells) + " |")
print("| **sum** | | " + " | ".join(f"**{x:.0f}**" for x in tot) + " |")
