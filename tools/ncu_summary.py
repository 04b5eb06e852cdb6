#!/usr/bin/env python
"""Summarise an .ncu-rep (read with `ncu -i ... --page raw --csv`) into per-kernel rows:
duration, achieved DRAM GB/s vs the measured HBM peak, tensor-pipe utilisation, L1/LSU pressure, top warp stalls.

    python tools/ncu_summary.py capture.ncu-rep [out.csv]
"""
import csv
import io
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rep = sys.argv[1]
out = sys.argv[2] if len(sys.argv) > 2 else None
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, data = rows[0], rows[1], rows[2:]
col = {h: i for i, h in enumerate(hdr)}
peak = 3350.0   # H100 SXM data sheet HBM3 GB/s, unless MEASURED_PEAKS.json is present
try:
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass


def get(r, name, default=float("nan")):
    i = col.get(name)
    if i is None or r[i] in ("", "n/a"):
        return default
    v = float(r[i].replace(",", ""))
    u = units[i]
    scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "ms": 1e-3, "us": 1e-6, "ns": 1e-9, "s": 1.0,
             "msecond": 1e-3, "usecond": 1e-6, "nsecond": 1e-9, "second": 1.0}.get(u)
    return v * scale if scale else v


stall_cols = [h for h in hdr if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
if not stall_cols:
    stall_cols = [h for h in hdr if h.startswith("smsp__average_warp_latency_issue_stalled_")]
fields = ["kernel", "grid", "ms", "dram_read_MB", "dram_write_MB", "dram_GBps", "frac_of_hbm_peak", "tensor_pipe_pct_active",
          "tensor_pipe_pct_elapsed", "sm_active_pct", "l1_lsu_pct", "lts_pct", "st_sectors_per_req", "ld_sectors_per_req",
          "regs", "top_stalls"]
res = []
for r in data:
    name = re.sub(r"\(.*", "", r[col["Kernel Name"]]).replace("lb::", "").replace("void ", "")
    t = get(r, "gpu__time_duration.sum")
    rd, wr = get(r, "dram__bytes_read.sum"), get(r, "dram__bytes_write.sum")
    stalls = sorted(((get(r, c, 0.0), c) for c in stall_cols), reverse=True)[:3]
    st_req, st_sec = get(r, "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum"), get(r, "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum")
    ld_req, ld_sec = get(r, "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum"), get(r, "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum")
    res.append({
        "kernel": name, "grid": r[col["Grid Size"]], "ms": round(t * 1e3, 4), "dram_read_MB": round(rd / 1e6, 2),
        "dram_write_MB": round(wr / 1e6, 2), "dram_GBps": round((rd + wr) / t / 1e9, 1),
        "frac_of_hbm_peak": round((rd + wr) / t / 1e9 / peak, 3),
        "tensor_pipe_pct_active": round(get(r, "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"), 1),
        "tensor_pipe_pct_elapsed": round(get(r, "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"), 1),
        "sm_active_pct": round(100 * get(r, "sm__cycles_active.avg") / max(get(r, "sm__cycles_elapsed.max"), 1), 1),
        "l1_lsu_pct": round(get(r, "l1tex__throughput.avg.pct_of_peak_sustained_active"), 1),
        "lts_pct": round(get(r, "lts__throughput.avg.pct_of_peak_sustained_elapsed"), 1),
        "st_sectors_per_req": round(st_sec / st_req, 1) if st_req == st_req and st_req else "",
        "ld_sectors_per_req": round(ld_sec / ld_req, 1) if ld_req == ld_req and ld_req else "",
        "regs": r[col["launch__registers_per_thread"]] if "launch__registers_per_thread" in col else "",
        "top_stalls": "; ".join(f"{c.split('stalled_')[1].split('_per_')[0]}={v:.2f}" for v, c in stalls),
    })
w = csv.DictWriter(open(out, "w", newline="") if out else sys.stdout, fieldnames=fields)
w.writeheader()
for x in res:
    w.writerow(x)
