"""Golden-vector cases of full (softmax) attention in the coarse and / or fine transformer (make_golden_full.py writes
them from the reference; the tests read them).  Kept apart from cases.CASES so that the tests parametrised over
CASES keep their parameter sets."""
from __future__ import annotations

import numpy as np

# 96 x 128 images: L = S = 192 coarse tokens, so the last 128-query tile of the coarse kernel is partial
FULL_CASES = [
    {"name": "full_ds_thr0", "n": 2, "hw0": (96, 128), "hw1": (96, 128), "thr": 0.0, "images": "smooth",
     "coarse_attention": "full", "fine_attention": "full"},
    {"name": "full_coarse_only", "n": 1, "hw0": (96, 128), "hw1": (96, 128), "thr": 0.0, "images": "smooth",
     "coarse_attention": "full", "fine_attention": "linear"},
    {"name": "full_fine_only", "n": 1, "hw0": (96, 128), "hw1": (96, 128), "thr": 0.0, "images": "smooth",
     "coarse_attention": "linear", "fine_attention": "full"},
    {"name": "full_ot", "n": 1, "hw0": (96, 128), "hw1": (96, 128), "thr": 0.0, "images": "smooth",
     "match_type": "sinkhorn", "coarse_attention": "full", "fine_attention": "full"},
    {"name": "full_unequal", "n": 1, "hw0": (96, 128), "hw1": (128, 104), "thr": 0.0, "images": "rand",
     "coarse_attention": "full", "fine_attention": "full"},
]

# Full-size parity cases of the GPU tests against the oracle (tests/util.oracle_forward_per_pair; precomputable
# on CPU with tools/precompute_oracle.py into the git-ignored tests/_oracle_cache/)
FULL_BASELINE_CASES = {
    "full_b2_640x480": {"name": "full_b2_640x480", "n": 2, "hw0": (480, 640), "hw1": (480, 640), "thr": 0.0,
                        "images": "smooth", "coarse_attention": "full", "fine_attention": "full"},
    "full_masked": {"name": "full_masked", "n": 2, "hw0": (512, 512), "hw1": (512, 512), "thr": 0.0, "images": "smooth",
                    "valid0": [(512, 384), (448, 512)], "valid1": [(384, 512), (512, 440)], "scales": True,
                    "coarse_attention": "full", "fine_attention": "full"},
}

# One reference FullAttention call with padding masks and finite inputs (valid rows pin the masked convention)
FA_MODULE_CASE = {"name": "fa_masked_module", "n": 2, "L": 150, "S": 131, "H": 8, "D": 32,
                  "valid_l": [150, 97], "valid_s": [101, 131]}


def build_fa_module_inputs(case=FA_MODULE_CASE):
    """-> q [n, L, H, D], k / v [n, S, H, D] float32 and bool masks [n, L], [n, S]."""
    rs = np.random.RandomState(5)
    n, L, S, H, D = case["n"], case["L"], case["S"], case["H"], case["D"]
    q = (rs.standard_normal((n, L, H, D)) * 1.5).astype(np.float32)
    k = (rs.standard_normal((n, S, H, D)) * 1.5).astype(np.float32)
    v = rs.standard_normal((n, S, H, D)).astype(np.float32)
    qm = np.zeros((n, L), bool)
    km = np.zeros((n, S), bool)
    for b in range(n):
        qm[b, : case["valid_l"][b]] = True
        km[b, : case["valid_s"][b]] = True
    return q, k, v, qm, km
