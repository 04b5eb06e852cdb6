"""CPU-side checks of the pair-count limit of one matching call (DESIGN.md §4.3): the coarse transformer's attention
kernels put the images of a pass in grid.z, whose CUDA limit is 65,535, so the C entries refuse larger counts before
any launch and the Python API raises ValueError before the backbone runs.  The GPU side (65,535 pairs run, bit for bit
against chunked calls) is tests/test_launch_limits_gpu.py."""
import ctypes as C

import pytest
import torch

import loftr_b200
import util
from loftr_b200 import _lib
from loftr_b200.loftr import MAX_PAIRS

LIMIT = 65535


def _model():
    return loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).eval()


@pytest.fixture
def no_stages(monkeypatch):
    return util.stages_unreachable(monkeypatch, _model())


def _pairs(n, hw=(8, 8)):
    return {"image0": torch.zeros(n, 1, *hw), "image1": torch.zeros(n, 1, *hw)}


def test_limit_is_the_grid_yz_limit():
    assert MAX_PAIRS == LIMIT


# ------------------------------------------------------------------------------------------------ C entries
def _refused(call, n, who):
    """`call(n)` with null buffers: at n = LIMIT + 1 it fails on the limit without launching; at LIMIT it passes the
    limit and stops at the buffers (there is no device here)."""
    lib = _lib.load()
    launches = lib.lb_launch_count()
    assert call(n) != 0
    msg = lib.lb_last_error()
    assert b"grid.z limit 65535" in msg and f"={n} ".encode() in msg and who in msg, msg
    assert lib.lb_launch_count() == launches
    assert call(LIMIT) != 0
    assert b"grid.z" not in lib.lb_last_error(), lib.lb_last_error()
    assert lib.lb_launch_count() == launches


def test_coarse_prep_refuses_more_than_65535_images():
    lib = _lib.load()
    buf = torch.zeros(64, dtype=torch.int32)
    p = buf.data_ptr()
    _refused(lambda n: lib.lb_coarse_prep(None, 1, None, n, 256, 1, 1, 1, 1, None, None, None, None), LIMIT + 1,
             b"coarse_prep: n_out")
    _refused(lambda n: lib.lb_coarse_prep_indexed(None, 1, None, p, n, 256, 1, 1, 1, 1, None, None, None, None),
             LIMIT + 1, b"coarse_prep: n_out")


@pytest.mark.parametrize("entry", ["lb_transformer_forward", "lb_transformer_forward_fp16"])
def test_coarse_transformer_refuses_more_than_65535_pairs(entry):
    fwd = getattr(_lib.load(), entry)

    def call(n, d_model=256):
        st = _lib.LbTransformerState(None, None, None, None, n, 1, 1, None)
        return fwd(None, None, 0, d_model, 8, C.byref(st), None, 0, None)

    _refused(call, LIMIT + 1, b"coarse transformer: n_groups")
    # the fine (window) transformer has no such limit: its groups are windows, in grid.x
    lib = _lib.load()
    assert call(10 * LIMIT, d_model=128) != 0 and b"grid.z" not in lib.lb_last_error(), lib.lb_last_error()


# ------------------------------------------------------------------------------------------------ Python API
def _bank(m):
    return util.host_bank(m, k=2)


def _calls(m, n):
    """Every matching call of the API on n pairs (n = 0 or more), with host inputs."""
    idx = torch.zeros(n, dtype=torch.int64)
    pts = torch.zeros(n, 1, 2)
    return {
        "forward": lambda: m(_pairs(n)),
        "forward_static": lambda: m.forward_static(_pairs(n)),
        "match_points": lambda: m.match_points(_pairs(n), pts),
        "match_features": lambda: m.match_features(_bank(m), idx, _bank(m), idx),
        "match_points_features": lambda: m.match_points_features(_bank(m), idx, _bank(m), idx, pts),
        "LocalFeatureTransformer": lambda: m.loftr_coarse(torch.zeros(n, 1, 256), torch.zeros(n, 1, 256)),
    }


@pytest.mark.parametrize("who", ["forward", "forward_static", "match_points", "match_features",
                                 "match_points_features", "LocalFeatureTransformer"])
def test_api_refuses_more_than_65535_pairs_before_the_backbone(no_stages, who):
    with pytest.raises(ValueError, match=rf"^{who}: 65536 pairs exceed the 65535 pairs of one call"):
        _calls(no_stages, LIMIT + 1)[who]()


@pytest.mark.parametrize("who", ["forward", "forward_static", "match_points", "match_features",
                                 "match_points_features", "LocalFeatureTransformer"])
def test_api_accepts_65535_pairs(no_stages, who):
    """65,535 pairs pass the count check: each call then stops at its next check (host tensors) or at a stage."""
    with pytest.raises((ValueError, RuntimeError, AssertionError)) as e:
        _calls(no_stages, LIMIT)[who]()
    assert "pairs exceed" not in str(e.value)


def test_fine_transformer_takes_any_window_count(no_stages):
    """The fine transformer's groups are windows (grid.x): the module refuses a host tensor, not the count."""
    with pytest.raises(RuntimeError, match="must live on a CUDA"):
        no_stages.loftr_fine(torch.zeros(LIMIT + 1, 1, 128), torch.zeros(LIMIT + 1, 1, 128))
