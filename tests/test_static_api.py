"""CPU-side checks of the sync-free forward and the graph-captured matcher: what they refuse before touching a device,
and the C-ABI fields they add."""
import ctypes

import pytest
import torch

import loftr_b200
from loftr_b200 import _lib


def _model(thr=0.0):
    return loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds", thr=thr)).eval()


def _data():
    return {"image0": torch.rand(1, 1, 64, 64), "image1": torch.rand(1, 1, 64, 64)}


def test_forward_static_rejects_host_inputs():
    with pytest.raises(ValueError, match="`image0` must already be a CUDA tensor"):
        _model().forward_static(_data())


def test_forward_static_rejects_data_dependent_configs_and_training():
    with pytest.raises(ValueError, match="thr >= 0"):
        _model(thr=-1.0).forward_static(_data())
    with pytest.raises(NotImplementedError):
        _model().train().forward_static(_data())
    with pytest.raises(ValueError, match="capacity"):
        _model().forward_static(_data(), capacity=0)


def test_captured_matcher_rejects_before_touching_a_device():
    with pytest.raises(ValueError, match="CUDA"):
        loftr_b200.CapturedMatcher(_model(), 1, (64, 64))
    with pytest.raises(ValueError, match="thr >= 0"):
        loftr_b200.CapturedMatcher(_model(thr=-1.0), 1, (64, 64))
    with pytest.raises(NotImplementedError):
        loftr_b200.CapturedMatcher(_model().train(), 1, (64, 64))


def test_device_count_fields_are_appended():
    """The live-count pointers come after every existing field, so older field offsets are unchanged."""
    for cls, name in ((_lib.LbTransformerState, "n_groups_live"), (_lib.LbFinePreprocessArgs, "M_live"),
                      (_lib.LbFineMatchArgs, "M_live")):
        assert cls._fields_[-1] == (name, ctypes.c_void_p)
        assert getattr(cls, name).offset == ctypes.sizeof(cls) - ctypes.sizeof(ctypes.c_void_p)
        assert getattr(cls(), name) is None   # NULL by default: the unbounded path
    assert _lib.load().lb_version() >= _lib.MIN_VERSION == 101
