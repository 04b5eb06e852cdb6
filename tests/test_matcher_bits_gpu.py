"""Exact output bits of the whole matcher (tests/golden/matcher_bits.npz, see make_golden_matcher_bits.py).

The cases launch every tensor-core kernel instantiation: the backbone's convolutions (gemm_split_kernel's convolution
mode, conv3x3_halo_kernel, the stem), the transformers' GEMMs with linear (kv_gemm_kernel) and full
(full_attn_wgmma_kernel) attention, both coarse matchings with and without the Sinkhorn prefilter, masked unequal-size
pairs, return_conf_matrix, the static path and the lb_gemm_split hook.  Further cases run the standalone fine
transformer's linear attention between windows of different sizes, with and without padding masks.  Every kernel is
deterministic, so every output must keep its bits, not merely stay within a tolerance."""
import os

import numpy as np
import pytest

import make_golden_matcher_bits as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "matcher_bits.npz")

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", G.NAMES)
def test_matcher_bits_unchanged(name):
    golden = np.load(GOLDEN)
    got = G.outputs(name)
    assert sorted(got) == list(golden[f"keys_{name}"]), "output keys changed"
    if name == G.FULL:
        for k, v in got.items():
            a, ref = v.cpu().numpy(), golden[f"full_{name}_{k}"]
            assert a.shape == ref.shape, f"{k}: shape {a.shape} vs {ref.shape}"
            assert a.tobytes() == ref.tobytes(), f"{k}: {np.count_nonzero(a != ref)} elements differ"
    changed = [k for k, v in got.items() if G.digest(v) != str(golden[f"sha_{name}_{k}"])]
    assert not changed, f"outputs changed: {changed}"
