"""Exact output bits of the backbone (tests/golden/backbone_bits.npz, see make_golden_backbone_bits.py).

conv3x3_halo_kernel splits its two consumer warpgroups by x-half of the 8 x 16 tile, and runs 196-channel outputs as
200-wide tiles.  Neither changes a summation order: every output element receives the same wgmma k-steps, in the same
order, as before.  So the feature maps must keep their bits, not merely stay within a tolerance, at batch 1 and 16 and
at grids that are not tile multiples.  (The NaN-filled workspace case of test_conv_halo_gpu.py runs the same 200-wide
tiles: channels 196..199 of the planes and columns 196..199 of the tile never reach an output.)"""
import os

import numpy as np
import pytest
import torch

import make_golden_backbone_bits as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "backbone_bits.npz")

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", G.SHAPES, ids=G.key)
def test_backbone_bits_unchanged(shape):
    golden = np.load(GOLDEN)
    fc, ff = G.backbone_bits(shape)
    k = G.key(shape)
    if shape == G.FULL:
        for got, name in ((fc, "feat_c"), (ff, "feat_f")):
            diff = (got.cpu() != torch.from_numpy(golden[f"{name}_{k}"])).nonzero()
            assert diff.numel() == 0, f"{name}: {diff.shape[0]} elements differ, first at {diff[0].tolist()}"
    assert G.digest(fc) == str(golden[f"sha_c_{k}"]), "coarse features changed"
    assert G.digest(ff) == str(golden[f"sha_f_{k}"]), "fine features changed"
