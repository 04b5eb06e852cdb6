"""Generate the full-attention golden vectors (tests/golden/full_cases.py) from the unmodified reference on the CPU in
fp32, the same way make_golden.py does for the linear cases.

    LOFTR_REFERENCE=<checkout> python tests/golden/make_golden_full.py   # writes tests/golden/full_*.npz, fa_*.npz
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
from full_cases import FA_MODULE_CASE, FULL_CASES, build_fa_module_inputs  # noqa: E402


def run_fa_module_case(case):
    """FullAttention.forward (linear_attention.py:56-81) with padding masks; padded rows come back NaN."""
    from src.loftr.loftr_module.linear_attention import FullAttention
    q, k, v, qm, km = build_fa_module_inputs(case)
    with torch.no_grad():
        out = FullAttention().eval()(*(torch.from_numpy(a) for a in (q, k, v, qm, km)))
    return {"out": out.numpy(), "q_mask": qm, "kv_mask": km}


def main():
    ref = ref_import.load_reference()
    torch.set_num_threads(8)
    for case in FULL_CASES:
        out = make_golden.run_case(ref, case)
        path = os.path.join(HERE, case["name"] + ".npz")
        np.savez_compressed(path, **out)
        print(f"{case['name']}: M={len(out['b_ids'])} (fp64 M={len(out['b_ids_f64'])}) conf.max={float(out['conf_max']):.4f} "
              f"-> {os.path.getsize(path) / 1024:.0f} KiB")
    out = run_fa_module_case(FA_MODULE_CASE)
    path = os.path.join(HERE, FA_MODULE_CASE["name"] + ".npz")
    np.savez_compressed(path, **out)
    print(f"{FA_MODULE_CASE['name']}: NaN rows={int(np.isnan(out['out']).any(axis=(2, 3)).sum())} "
          f"-> {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
