"""loftr_b200 -- H100-native LoFTR matching engine; drop-in for `from src.loftr import LoFTR, default_cfg`."""
from .config import default_cfg, get_cfg
from .geometry import estimate_geometry
from .loftr import CapturedMatcher, ImageFeatures, LoFTR
from .preprocess import PreparedImages, prepare_images, prepare_pairs, rotation_candidates, target_size, warp_images

__all__ = ["CapturedMatcher", "ImageFeatures", "LoFTR", "PreparedImages", "default_cfg", "estimate_geometry", "get_cfg",
           "prepare_images", "prepare_pairs", "rotation_candidates", "target_size", "warp_images"]
