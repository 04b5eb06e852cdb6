"""Import the UNMODIFIED reference (a zju3dv/LoFTR checkout named by $LOFTR_REFERENCE) for oracle validation and
golden-vector generation -- TEST INFRASTRUCTURE, only usable where such a checkout exists; the tests themselves read
the stored golden vectors and never need it.

The reference needs three modules that are not installed / not shipped:
  * kornia (pinned 0.4.1): only `dsnt.spatial_expectation2d` and `create_meshgrid` are on the hot path
    (fine_matching.py:5-6,49-50) -> 10-line stand-ins with the documented semantics; the evaluation metrics
    (src/utils/metrics.py:6-7) additionally use `epipolar.numeric.cross_product_matrix` and
    `conversions.convert_points_to_homogeneous` -> two more stand-ins.
  * yacs: `CfgNode` is used as an attribute dict (cvpr_ds_config.py:1-9) -> a dict subclass.
  * src/loftr/utils/superglue.py: deliberately absent from the reference (README.md:63-74); the pinned
    submodule copy third_party/SuperGluePretrainedNetwork/models/superglue.py is registered under that
    name (used as an ORACLE only; its licence forbids copying it).
Nothing from the reference is copied into this repository.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

REF_ROOT = os.environ.get("LOFTR_REFERENCE", "")


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "src", "loftr"))


def _install_stubs():
    import torch

    if "kornia" not in sys.modules:
        def create_meshgrid(height, width, normalized_coordinates=True, device=None, dtype=torch.float32):
            xs = torch.linspace(0, width - 1, width, device=device, dtype=dtype)
            ys = torch.linspace(0, height - 1, height, device=device, dtype=dtype)
            if normalized_coordinates:
                xs = (xs / (width - 1) - 0.5) * 2
                ys = (ys / (height - 1) - 0.5) * 2
            gy, gx = torch.meshgrid(ys, xs, indexing="ij")
            return torch.stack([gx, gy], dim=-1).unsqueeze(0)  # [1, H, W, 2] (x, y)

        def spatial_expectation2d(inp, normalized_coordinates=True):
            b, n, h, w = inp.shape
            grid = create_meshgrid(h, w, normalized_coordinates, inp.device, inp.dtype)
            px = grid[..., 0].reshape(1, 1, -1)
            py = grid[..., 1].reshape(1, 1, -1)
            flat = inp.reshape(b, n, -1)
            ex = (flat * px).sum(-1, keepdim=True)
            ey = (flat * py).sum(-1, keepdim=True)
            return torch.cat([ex, ey], -1)  # [B, N, 2]

        def cross_product_matrix(x):   # kornia.geometry.epipolar.numeric: [..., 3] -> [..., 3, 3] skew-symmetric
            z = torch.zeros_like(x[..., 0])
            return torch.stack([torch.stack([z, -x[..., 2], x[..., 1]], -1), torch.stack([x[..., 2], z, -x[..., 0]], -1),
                                torch.stack([-x[..., 1], x[..., 0], z], -1)], -2)

        def convert_points_to_homogeneous(points):   # kornia.geometry.conversions: append a 1
            return torch.nn.functional.pad(points, [0, 1], "constant", 1.0)

        kornia = types.ModuleType("kornia")
        geometry = types.ModuleType("kornia.geometry")
        epipolar = types.ModuleType("kornia.geometry.epipolar")
        numeric = types.ModuleType("kornia.geometry.epipolar.numeric")
        conversions = types.ModuleType("kornia.geometry.conversions")
        numeric.cross_product_matrix = cross_product_matrix
        epipolar.numeric = numeric
        conversions.convert_points_to_homogeneous = convert_points_to_homogeneous
        geometry.epipolar, geometry.conversions = epipolar, conversions
        subpix = types.ModuleType("kornia.geometry.subpix")
        dsnt = types.ModuleType("kornia.geometry.subpix.dsnt")
        utils = types.ModuleType("kornia.utils")
        grid = types.ModuleType("kornia.utils.grid")
        dsnt.spatial_expectation2d = spatial_expectation2d
        subpix.dsnt = dsnt
        geometry.subpix = subpix
        grid.create_meshgrid = create_meshgrid
        utils.grid = grid
        utils.create_meshgrid = create_meshgrid
        kornia.geometry, kornia.utils = geometry, utils
        for name, mod in [("kornia.geometry.epipolar", epipolar), ("kornia.geometry.epipolar.numeric", numeric),
                          ("kornia.geometry.conversions", conversions)]:
            sys.modules[name] = mod
        for name, mod in [("kornia", kornia), ("kornia.geometry", geometry), ("kornia.geometry.subpix", subpix),
                          ("kornia.geometry.subpix.dsnt", dsnt), ("kornia.utils", utils), ("kornia.utils.grid", grid)]:
            sys.modules[name] = mod

    if "yacs" not in sys.modules:
        class CfgNode(dict):
            def __getattr__(self, k):
                try:
                    return self[k]
                except KeyError as e:
                    raise AttributeError(k) from e

            def __setattr__(self, k, v):
                self[k] = v

            def clone(self):
                import copy
                return copy.deepcopy(self)

        yacs = types.ModuleType("yacs")
        cfgmod = types.ModuleType("yacs.config")
        cfgmod.CfgNode = CfgNode
        yacs.config = cfgmod
        sys.modules["yacs"], sys.modules["yacs.config"] = yacs, cfgmod


def load_reference():
    """Returns the reference's `src.loftr` package (LoFTR, default_cfg) with the stubs above installed."""
    if not available():
        raise RuntimeError(f"reference not found under {REF_ROOT}")
    _install_stubs()
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    name = "src.loftr.utils.superglue"
    if name not in sys.modules:
        import src.loftr.utils  # noqa: F401  (parent package first)
        path = os.path.join(REF_ROOT, "third_party", "SuperGluePretrainedNetwork", "models", "superglue.py")
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
    import src.loftr as ref
    return ref


def load_reference_metrics():
    """The reference's src/utils/metrics.py module (evaluation harness; needs cv2 and loguru, both installed)."""
    load_reference()
    import numpy as np
    if not hasattr(np, "bool"):       # metrics.py:128 uses the alias removed in numpy 1.24
        np.bool = bool
    if not hasattr(np, "trapz"):      # metrics.py:159; numpy >= 2.4 drops it
        np.trapz = np.trapezoid
    import src.utils.metrics as m
    return m
