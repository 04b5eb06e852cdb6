"""The timing protocol the A/B tools in tools/ share, so that their numbers stay comparable with each other and with
BASELINE.md.  A tool supplies its workload; this module supplies the GPU check, the card label, the L2 flush, the
CUDA-event timing, the alternation of arms and the kernel-tag pass.
"""
import subprocess
import sys

import torch

from loftr_b200 import _lib

_flush_buf = None


def require_gpu(tool):
    """cuda:0, or exit: a GPU timing has no CPU fallback."""
    if not torch.cuda.is_available():
        sys.exit(f"{tool}: no CUDA device (this measurement needs an H100)")
    return torch.device("cuda:0")


def gpu_label():
    """The card's name and power limit, which belong beside every number measured on it (read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], check=True,
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the numbers stay valid; say where the label is missing
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({type(e).__name__})"}


def stats(v, nd=3):
    """min, upper median and max of v, rounded to nd decimals."""
    v = sorted(v)
    return {"min": round(v[0], nd), "median": round(v[len(v) // 2], nd), "max": round(v[-1], nd)}


def _flush_l2():
    """Write a 256 MiB buffer (allocated on first use, then kept) so that the 50 MB L2 holds nothing of the last call."""
    global _flush_buf
    if _flush_buf is None:
        _flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    _flush_buf.zero_()


def timed(fn, flush=True):
    """(fn(), ms between CUDA events recorded around it), after an untimed L2 flush when `flush`."""
    if flush:
        _flush_l2()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def alternate(arms, reps, warmup, flush=True):
    """`warmup` untimed rounds over every arm, then `reps` timed rounds, each calling the arms {name: fn} in order, so
    every arm sees the same clocks and neighbours.  -> ({name: [ms per round]}, {name: output of its last call})."""
    for _ in range(warmup):
        for fn in arms.values():
            timed(fn, flush)
    ms, last = {name: [] for name in arms}, {}
    for _ in range(reps):
        for name, fn in arms.items():
            last[name], t = timed(fn, flush)
            ms[name].append(t)
    return ms, last


def tag_ms(fn, runs=1, flush=False):
    """{tag: (total ms, launches)} of the library's tagged kernels over `runs` calls of fn, with CUDA events around
    every tagged launch; in a pass of its own, since those events slow the host."""
    _lib.timing_enable(True)
    try:
        for _ in range(runs):
            if flush:
                _flush_l2()
            fn()
        return _lib.timing_collect()
    finally:
        _lib.timing_enable(False)
