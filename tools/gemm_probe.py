#!/usr/bin/env python
"""Main-loop vs epilogue probe of gemm_split_kernel through the lb_gemm_split test hook: the same problem is timed
with the normal store epilogue, with TMEM loads only, and with a null epilogue (LOFTR_B200_PROBE_NULL_EPI = 0/2/1,
read per call).  Shapes are the coarse-transformer GEMMs of the bench workload (76800 rows)."""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from loftr_b200 import _lib  # noqa: E402
from loftr_b200.loftr import split_planes, _stream  # noqa: E402

lib = _lib.load()
dev = "cuda:0"
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
for (m, n, k) in [(76800, 256, 256), (76800, 768, 256), (76800, 512, 512), (76800, 256, 512), (38400, 256, 256), (4800 * 3 + 77, 256, 256)]:
    a = torch.randn(m, k, device=dev)
    w = torch.randn(n, k, device=dev)
    ah, al = split_planes(a)
    wh, wl = split_planes(w)
    out = torch.empty(m, n, dtype=torch.float32, device=dev)
    res = {}
    outs = {}
    for mode, name in ((0, "store"), (2, "tmem_ld_only"), (1, "null")):
        os.environ["LOFTR_B200_PROBE_NULL_EPI"] = str(mode)
        ts = []
        for it in range(6):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(lib.lb_gemm_split(ah.data_ptr(), al.data_ptr(), k, 0, wh.data_ptr(), wl.data_ptr(), k, 0,
                                         out.data_ptr(), n, 0, 1, m, n, k, _stream(out)))
            e1.record()
            torch.cuda.synchronize()
            if it >= 2:
                ts.append(e0.elapsed_time(e1))
        res[name] = sum(ts) / len(ts)
        if mode == 0:
            outs[mode] = out.clone()
    ref = (a.double() @ w.double().T)
    same = f"{float((outs[0].double() - ref).abs().max() / ref.abs().max()):.2e}"
    fl = 2.0 * m * n * k * 3
    print(f"M={m} N={n} K={k}: " + "  ".join(f"{kk} {v * 1e3:7.1f} us ({fl / v / 1e9:6.0f} TF/s issued)" for kk, v in res.items()) + f"  rel err vs fp64: {same}", flush=True)
os.environ["LOFTR_B200_PROBE_NULL_EPI"] = "0"
