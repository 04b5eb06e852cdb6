"""Image front end (`prepare_images`, DESIGN.md §14) against the host glue it replaces, alternating in one process.

Workloads: 16 uint8 frames 968x1296 -> 640x480 (a batch of 8 ScanNet pairs) and 8 frames 1200x1600 -> longer edge 832,
square-padded (MegaDepth style), uniform-random pixels from a fixed seed.  Arms, per workload and per step:
  host_glue     per image cv2.resize + float + / 255 (+ zero padding and the 1/8 mask) on one host thread, stacked
                into a pinned fp32 batch and copied to the device; reported as absent when cv2 cannot be imported;
  gpu_front_end the uint8 frames copied from pinned memory to the device, then `prepare_images` on them.
Reported: ms per batch (host clock around a device synchronise; min / median / max), the kernel's own time from the
`preprocess` timing tag in a pass of its own (a 256 MiB buffer written before every launch), the bytes the kernel
reads and writes computed from the shapes (`kernel_bytes`), the resulting GB/s next to the 3.35 TB/s HBM3 data-sheet figure (the kernel is HBM-bound; the share is of a figure for a 700 W card), and
the GPU name and power limit.  Prints one JSON line; fails without a CUDA device.

    python tools/preprocess_bench.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import loftr_b200  # noqa: E402
from measure import gpu_label, require_gpu, stats, tag_ms  # noqa: E402

HBM_DATASHEET_GBPS = 3350.0
# (name, frames, (h, w), resize, pad_to)
WORKLOADS = [
    ("16x968x1296_to_480x640", 16, (968, 1296), (640, 480), None),
    ("8x1200x1600_to_832_square", 8, (1200, 1600), 832, "square"),
]


def kernel_bytes(n, h, w, h_new, w_new, H, W, masked):
    """The least one launch moves through HBM: every source byte its taps touch, once (two rows and two columns per
    output row and column, so all of the image up to a 2x reduction per axis), the fp32 canvas and the mask."""
    read = n * min(h, 2 * h_new) * min(w, 2 * w_new)
    return read + n * H * W * 4 + (n * (H // 8) * (W // 8) if masked else 0)


def run(name, n, hw, resize, pad_to, steps, warmup, dev):
    h, w = hw
    rs = np.random.RandomState(7)
    frames = [rs.randint(0, 256, (h, w)).astype(np.uint8) for _ in range(n)]
    w_new, h_new = loftr_b200.target_size(w, h, resize)
    H, W = (max(h_new, w_new),) * 2 if pad_to == "square" else (h_new, w_new)
    try:
        import cv2
    except ImportError:
        cv2 = None
    pinned_f32 = torch.empty((n, 1, H, W), dtype=torch.float32, pin_memory=True)
    pinned_u8 = torch.empty((n, h, w), dtype=torch.uint8, pin_memory=True)

    masks = np.zeros((n, H // 8, W // 8), bool)

    def host_glue():
        batch = pinned_f32.numpy()
        for k, f in enumerate(frames):
            img = cv2.resize(f, (w_new, h_new))
            if pad_to is not None:
                batch[k, 0] = 0
                full = np.zeros((H, W), bool)
                full[:h_new, :w_new] = True
                masks[k] = full[::8, ::8]
            batch[k, 0, :h_new, :w_new] = img.astype(np.float32) / 255
        return pinned_f32.to(dev, non_blocking=True)

    def gpu_front_end():
        for k, f in enumerate(frames):   # what a decoder would do: write the frame into pinned memory
            pinned_u8[k] = torch.from_numpy(f)
        return loftr_b200.prepare_images(pinned_u8.to(dev, non_blocking=True), resize=resize, pad_to=pad_to).image

    arms = {"gpu_front_end": gpu_front_end}
    if cv2 is not None:
        arms["host_glue"] = host_glue
    for _ in range(warmup):
        for fn in arms.values():
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(steps):
        for k, fn in arms.items():   # alternate: both arms see the same clocks and neighbours
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t0) * 1e3)

    dev_frames = pinned_u8.to(dev)
    # flushed: the frames would otherwise stay in the 50 MB L2 from one launch to the next
    k_ms, k_n = tag_ms(lambda: loftr_b200.prepare_images(dev_frames, resize=resize, pad_to=pad_to), runs=steps,
                       flush=True)["preprocess"]
    kernel_ms = k_ms / k_n
    nbytes = kernel_bytes(n, h, w, h_new, w_new, H, W, pad_to is not None)
    gbps = nbytes / (kernel_ms * 1e-3) / 1e9
    res = {"workload": name, "frames": n, "source_hw": [h, w], "valid_hw": [h_new, w_new], "canvas_hw": [H, W],
           "gpu_front_end_ms": stats(ms["gpu_front_end"]),
           "host_glue_ms": stats(ms["host_glue"]) if cv2 is not None else "absent (cv2 cannot be imported)",
           "h2d_bytes": {"gpu_front_end": n * h * w, "host_glue": n * H * W * 4},
           "kernel_ms": round(kernel_ms, 4), "kernel_launches": k_n, "kernel_bytes": nbytes,
           "kernel_gbps": round(gbps, 1), "share_of_hbm_datasheet": round(gbps / HBM_DATASHEET_GBPS, 3)}
    if cv2 is not None:
        res["cv2_version"], res["cv2_threads"] = cv2.__version__, cv2.getNumThreads()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = require_gpu("preprocess_bench")
    out = {"tool": "preprocess_bench", "steps": args.steps, **gpu_label(), "bound": "HBM",
           "hbm_datasheet_gbps": HBM_DATASHEET_GBPS,
           "workloads": [run(*w, args.steps, args.warmup, dev) for w in WORKLOADS]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
