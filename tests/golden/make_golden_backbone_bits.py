"""Record the exact output bits of lb_backbone_forward (tests/golden/backbone_bits.npz) for
tests/test_conv_halo_rowsplit_gpu.py: the SHA-256 of the coarse and fine feature maps at each shape of SHAPES, and both
maps in full for the smallest one.  Changing which warpgroup issues a convolution's MMAs, or the width of its output
tile, must not change these bits; a change to any summation order must regenerate them (and say so).  Needs an H100;
LOFTR_B200_LIB selects the build that defines the reference bits.

    LOFTR_B200_LIB=<variant> python tests/golden/make_golden_backbone_bits.py [OUT.npz]
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

# (images, height, width): grids that are not multiples of the 8 x 16 output tile at 1/2, 1/4 and 1/8, and the bench size
SHAPES = [(1, 16, 16), (16, 16, 16), (1, 136, 200), (16, 136, 200), (1, 88, 72), (16, 88, 72), (1, 480, 640),
          (16, 480, 640)]
FULL = (1, 16, 16)   # stored in full as well
SEED = 21


def key(shape):
    return "x".join(str(v) for v in shape)


def digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def backbone_bits(shape, dev="cuda:0"):
    """-> (feat_c, feat_f) of lb_backbone_forward on the test weights and a seeded image batch of `shape`."""
    import backbone_ref as B
    import util
    from cases import CASES
    from loftr_b200.loftr import TensorCoreBackbone
    model, _, _ = util.build_model(dict(CASES[0]), dev)
    return B.backbone_forward(TensorCoreBackbone(model.backbone), B.image(shape, SEED, dev))[1:]


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "backbone_bits.npz")
    out = {}
    for shape in SHAPES:
        fc, ff = backbone_bits(shape)
        out[f"sha_c_{key(shape)}"] = np.array(digest(fc))
        out[f"sha_f_{key(shape)}"] = np.array(digest(ff))
        if shape == FULL:
            out[f"feat_c_{key(shape)}"] = fc.cpu().numpy()
            out[f"feat_f_{key(shape)}"] = ff.cpu().numpy()
        print(key(shape), out[f"sha_c_{key(shape)}"], out[f"sha_f_{key(shape)}"], flush=True)
    np.savez_compressed(out_path, **out)
    print(f"-> {out_path} ({os.path.getsize(out_path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
