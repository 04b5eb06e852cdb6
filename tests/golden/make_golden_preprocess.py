"""Golden vectors for the image front end (DESIGN.md §14): runs the UNMODIFIED reference functions of
src/utils/dataset.py (get_resized_wh, get_divisible_wh, read_megadepth_gray with pad_bottom_right, read_scannet_gray),
the 1/8 mask interpolation of src/datasets/megadepth.py:121-124 and cv2.cvtColor on the seeded inputs of
preprocess_cases.py and stores the outputs in tests/golden/preprocess_cases.npz.  Authoring container only: needs the
reference checkout ($LOFTR_REFERENCE) and OpenCV.  The reference module imports h5py (depth maps, not used here), which
is absent: an empty stand-in is registered.  Its image reader is pointed at the in-memory inputs; nothing is copied.

    LOFTR_REFERENCE=/path/to/LoFTR python tests/golden/make_golden_preprocess.py
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import ref_import  # noqa: E402
from preprocess_cases import GREY_HW, GREY_SEED, IMAGE_CASES, SIZE_CASES, image  # noqa: E402


def load_reference_dataset_utils():
    if not ref_import.available():
        raise RuntimeError(f"reference not found under {ref_import.REF_ROOT}")
    sys.modules.setdefault("h5py", types.ModuleType("h5py"))
    if ref_import.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REF_ROOT)
    import src.utils.dataset as D
    return D


def main():
    import cv2
    D = load_reference_dataset_utils()
    out = {"cv2_version": np.asarray(cv2.__version__)}
    sizes = []
    for w, h, resize, df in SIZE_CASES:
        wh = resize if isinstance(resize, tuple) else D.get_resized_wh(w, h, resize)
        sizes.append(D.get_divisible_wh(*wh, df))
    out["sizes"] = np.asarray(sizes, np.int64)

    inputs = {name: image(seed, h, w) for name, (seed, h, w, _, _) in IMAGE_CASES.items()}
    D.imread_gray = lambda path, augment_fn=None, client=None: inputs[path]   # the reader's only file access
    for name, (_, h, w, resize, df) in IMAGE_CASES.items():
        if name.startswith("md_"):
            img, mask, scale = D.read_megadepth_gray(name, resize, df, True, None)
            mask_c = F.interpolate(mask[None, None].float(), scale_factor=0.125, mode="nearest",
                                   recompute_scale_factor=False)[0, 0].bool()
            out[name + "_mask"] = mask_c.numpy()
            out[name + "_scale"] = scale.numpy()
        elif name.startswith("sc_"):
            img = D.read_scannet_gray(name, resize, None)
        else:
            w_new, h_new = D.get_divisible_wh(*D.get_resized_wh(w, h, resize), df)
            img = torch.from_numpy(cv2.resize(inputs[name], (w_new, h_new))).float()[None] / 255
        levels = np.rint(img[0].numpy().astype(np.float64) * 255)
        assert np.abs(levels / 255 - img[0].numpy()).max() < 1e-6
        out[name + "_levels"] = levels.astype(np.uint8)     # cv2.resize output, zero-padded for md_*

    rgb = image(GREY_SEED, *GREY_HW, channels=3)
    out["grey_from_rgb"] = cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY)
    out["grey_from_bgr"] = cv2.cvtColor(rgb, cv2.COLOR_BGR2GRAY)
    path = os.path.join(HERE, "preprocess_cases.npz")
    np.savez_compressed(path, **out)
    print({k: v.shape for k, v in out.items()})
    print("->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
