"""Exhaustive pair list over a small image set: `matcher(batch)` against a feature bank (`extract_features` once, then
`match_features` per batch), alternating in one process.

16 seeded 640x480 images, all 120 pairs (i < j) in 15 batches of 8, indoor_ds at thr 0 with seeded weights and the
tensor-core backbone (the default).  One repetition runs the whole list both ways:
  plain: 15 steps of `matcher(batch)` on the stacked images of 8 pairs (the backbone sees 16 images per step);
  bank:  one `extract_features` step on the 16 images, then 15 steps of `match_features` on the same 8-pair batches.
A 256 MiB buffer is written before every step (untimed; flushes the 50 MB L2) and every step is timed with CUDA events.
Reported: ms per step (min / median / max over steps), ms and pairs/s per list (min / median / max over repetitions),
the share of the plain step spent in the backbone's convolutions (`backbone_conv` kernel timing tag, from a separate
profiled pass; the 7x7 stem is not tagged), and whether both produced bit-identical outputs for every batch.  Prints
one JSON line with the GPU name and power limit.

    python tools/pair_list_bench.py [--reps 5] [--warmup 1]
"""
import argparse
import itertools
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import loftr_b200  # noqa: E402
from measure import gpu_label, require_gpu, stats, tag_ms, timed  # noqa: E402

N_IMAGES, H, W, BATCH = 16, 480, 640, 8
KEYS = ["b_ids", "i_ids", "j_ids", "gt_mask", "m_bids", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f",
        "expec_f"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    dev = require_gpu("pair_list_bench")
    torch.manual_seed(0)
    model = loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=0.0)).eval().to(dev)
    g = torch.Generator().manual_seed(1000)
    images = torch.rand(N_IMAGES, 1, H, W, generator=g).to(dev)
    pairs = torch.tensor(list(itertools.combinations(range(N_IMAGES), 2)), device=dev)
    batches = [(pairs[s:s + BATCH, 0].contiguous(), pairs[s:s + BATCH, 1].contiguous())
               for s in range(0, len(pairs), BATCH)]

    def plain_step(i0, i1):
        d = {"image0": images[i0], "image1": images[i1]}
        model(d)
        return d

    def run_plain():
        outs, ms = [], []
        for i0, i1 in batches:
            d, t = timed(lambda: plain_step(i0, i1))
            outs.append(d)
            ms.append(t)
        return outs, ms

    def run_bank():
        bank, t_ext = timed(lambda: model.extract_features(images))
        outs, ms = [], []
        for i0, i1 in batches:
            d, t = timed(lambda: model.match_features(bank, i0, bank, i1))
            outs.append(d)
            ms.append(t)
        del bank
        return outs, ms, t_ext

    for _ in range(args.warmup):
        run_plain()
        run_bank()
    plain_ms, bank_ms, extract_ms, plain_list_ms, bank_list_ms = [], [], [], [], []
    identical, matches = True, 0
    for _ in range(args.reps):   # alternate: both see the same clocks and neighbours
        p_out, p_ms = run_plain()
        b_out, b_ms, t_ext = run_bank()
        plain_ms += p_ms
        bank_ms += b_ms
        extract_ms.append(t_ext)
        plain_list_ms.append(sum(p_ms))
        bank_list_ms.append(t_ext + sum(b_ms))
        for p, b in zip(p_out, b_out):
            identical &= all(torch.equal(p[k], b[k]) for k in KEYS)
        matches = sum(int(p["b_ids"].shape[0]) for p in p_out)
        del p_out, b_out

    # backbone share of the plain step: per-launch events around the tagged kernels, in a pass of its own
    prof_ms = []
    tags = tag_ms(lambda: prof_ms.extend(run_plain()[1]))
    conv_ms = tags.get("backbone_conv", (0.0, 0))[0]

    n_pairs = len(pairs)
    res = {"tool": "pair_list_bench", **gpu_label(), "images": N_IMAGES, "hw": [H, W], "pairs": n_pairs,
           "batch": BATCH, "reps": args.reps, "matches_per_list": matches, "outputs_identical": bool(identical),
           "plain_ms_per_step": stats(plain_ms), "bank_match_ms_per_step": stats(bank_ms),
           "bank_extract_ms": stats(extract_ms),
           "plain_ms_per_list": stats(plain_list_ms), "bank_ms_per_list": stats(bank_list_ms),
           "plain_pairs_per_s": stats([n_pairs * 1e3 / t for t in plain_list_ms]),
           "bank_pairs_per_s": stats([n_pairs * 1e3 / t for t in bank_list_ms]),
           "backbone_conv_share_of_plain_step": round(conv_ms / sum(prof_ms), 4),
           "extract16_over_plain_step_median": round(stats(extract_ms)["median"] / stats(plain_ms)["median"], 4),
           "l2": "256 MiB buffer written before every step"}
    print(json.dumps(res))
    assert identical, "match_features and matcher(batch) disagree"


if __name__ == "__main__":
    main()
