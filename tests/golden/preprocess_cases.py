"""Inputs of the image front-end goldens (tests/golden/preprocess_cases.npz), regenerated from seeds; only the outputs
of the reference pipeline and of OpenCV are stored (make_golden_preprocess.py)."""
import numpy as np

# (w, h, resize, df): int = longer edge, pair = literal (w, h).  Rows 0-3 put w*scale or h*scale exactly on .5 (Python's
# round goes to the even neighbour: 2.5 -> 2, 3.5 -> 4, 12.5 -> 12, 37.5 -> 38); the later ones are truncated by df.
SIZE_CASES = [
    (5, 10, 5, 1), (7, 10, 5, 1), (25, 50, 25, 1), (100, 75, 50, 1),
    (1296, 968, (640, 480), 8), (1600, 1200, 832, 8), (1200, 1600, 832, 8), (777, 1001, 832, 8), (400, 300, 832, 8),
    (1001, 777, 840, 8), (640, 480, None, 8), (645, 487, None, 8), (100, 36, 50, 8), (333, 500, 200, 16),
    (1920, 1080, 1200, 8), (9, 9, 64, 8),
]

# name -> (seed, h, w, resize, df).  "md_*" run through read_megadepth_gray with padding (square canvas, mask, scale);
# "sc_*" through read_scannet_gray (literal size); "id_*" keeps its size.
IMAGE_CASES = {
    "md_down": (11, 300, 400, 208, 8),
    "md_up": (12, 60, 45, 128, 8),
    "md_odd": (13, 101, 77, 96, 8),
    "md_wide": (14, 90, 250, 120, 8),
    "sc_down": (15, 242, 324, (160, 120), 8),
    "id_same": (16, 64, 80, None, 8),
}
GREY_SEED, GREY_HW = 21, (64, 96)


def image(seed, h, w, channels=1):
    rs = np.random.RandomState(seed)
    return rs.randint(0, 256, (h, w) if channels == 1 else (h, w, channels)).astype(np.uint8)
