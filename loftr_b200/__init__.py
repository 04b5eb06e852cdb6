"""loftr_b200 -- H100-native LoFTR matching engine; drop-in for `from src.loftr import LoFTR, default_cfg`."""
from .config import default_cfg, get_cfg
from .loftr import CapturedMatcher, LoFTR

__all__ = ["CapturedMatcher", "LoFTR", "default_cfg", "get_cfg"]
