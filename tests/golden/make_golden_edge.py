"""Generate the edge-configuration golden vectors (tests/golden/edge_cases.py) from the unmodified reference on the CPU
in fp32 (plus its float64 run), the same way make_golden.py does for the base cases.

    LOFTR_REFERENCE=<checkout> python tests/golden/make_golden_edge.py   # writes tests/golden/edge_*.npz
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from oracle import ref_import  # noqa: E402
import make_golden  # noqa: E402
from edge_cases import EDGE_CASES, build_edge_cfg  # noqa: E402


def main():
    ref = ref_import.load_reference()
    torch.set_num_threads(8)
    make_golden.build_cfg = build_edge_cfg   # run_case builds the model from the case's config
    for case in EDGE_CASES:
        out = make_golden.run_case(ref, case)
        path = os.path.join(HERE, case["name"] + ".npz")
        np.savez_compressed(path, **out)
        print(f"{case['name']}: M={len(out['b_ids'])} (fp64 M={len(out['b_ids_f64'])}) W={out['fine_pre0'].shape[1]} "
              f"-> {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
