"""Golden-vector cases of configurations at the edges of what the kernels accept (make_golden_edge.py writes them from
the reference; the tests read them).  Kept apart from cases.CASES so that the tests parametrised over CASES keep their
parameter sets."""
from __future__ import annotations

from cases import build_cfg

# fine_window_size = 3: 9-row windows, refinement grid step 2 / (W - 1) = 1, W // 2 = 1
EDGE_CASES = [
    {"name": "edge_w3_ds_thr0", "n": 2, "hw0": (96, 128), "hw1": (96, 128), "thr": 0.0, "images": "smooth",
     "fine_window_size": 3},
]


def build_edge_cfg(case):
    cfg = build_cfg(case)
    cfg["fine_window_size"] = case.get("fine_window_size", 5)
    return cfg
