"""CPU-side checks of the feature-bank matcher (`LoFTR.extract_features` / `LoFTR.match_features`): the library
version guard and what is refused before any device work."""
import pytest
import torch

import loftr_b200
import util
from loftr_b200 import _lib


def _model():
    return loftr_b200.LoFTR(loftr_b200.get_cfg("indoor_ds")).eval()


def test_match_features_refuses_an_older_library(monkeypatch):
    util.old_library(monkeypatch, 103)
    assert _lib.FEATURE_BANK_VERSION == 104
    with pytest.raises(RuntimeError, match=r"version 104 or newer.*is version 103"):
        _model().match_features(None, None, None, None)


def test_indexed_entry_points_are_bound():
    lib = _lib.load()
    assert lib.lb_version() >= _lib.FEATURE_BANK_VERSION
    for name in ("lb_coarse_prep_indexed", "lb_fine_preprocess_indexed"):
        assert _lib.SIGNATURES[name][1] == getattr(lib, name).argtypes


def test_extract_features_refuses_host_images_and_training():
    with pytest.raises(RuntimeError, match="CUDA"):
        _model().extract_features(torch.rand(2, 1, 64, 64))
    with pytest.raises(NotImplementedError):
        _model().train().extract_features(torch.rand(2, 1, 64, 64))
    with pytest.raises(NotImplementedError):
        _model().train().match_features(None, None, None, None)
