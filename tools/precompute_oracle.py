#!/usr/bin/env python
"""Precompute the numpy-oracle outputs (+ fp64 near-tie statistics) of the full-size BASELINE.json parity cases on
CPU into tests/_oracle_cache/ (git-ignored), so that the GPU machine
spends its time on the engine, not on the CPU oracle.  A missing / stale entry is recomputed by the tests.

    python tools/precompute_oracle.py [case ...]
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import util  # noqa: E402
from cases import BASELINE_CASES  # noqa: E402
from full_cases import FULL_BASELINE_CASES  # noqa: E402

cases = {**BASELINE_CASES, **FULL_BASELINE_CASES}   # the second: full (softmax) attention, test_full_attention_gpu.py
for name in sys.argv[1:] or list(cases):
    t0 = time.time()
    res, gold = util.oracle_forward_per_pair(cases[name], "cpu", adjudicate=name != "b8thr")
    print(f"{name}: {len(res['b_ids'])} matches, adjudication stats: {gold is not None}, {time.time() - t0:.0f} s", flush=True)
