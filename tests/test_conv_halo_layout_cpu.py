"""Address arithmetic of conv3x3_halo_kernel (loftr_b200/csrc/conv_halo.cuh), replayed in Python: the no-swizzle
wgmma descriptors over the shared-memory halo [8-channel chunk][halo pixel][16 bytes] must read exactly the im2col
operand of the 8 x 16 output tile for all nine taps, both x-halves, every k-step, partial edge tiles and the
16-channel remainder halo; the accumulator row -> tile pixel map must be the inverse of the kernel's staging."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "loftr_b200", "csrc", "conv_halo.cuh")).read()
CHUNK = int(re.search(r"constexpr int kHaloChunkBytes = (\d+);", SRC).group(1))
HW, HH, TW, TH = 18, 10, 16, 8
LBO, SBO = CHUNK, HW * 16


def load_halo(x, batch, ty, tx, c0, chunks):
    """What the producer's TMA boxes write: (chunk, halo pixel, 8 channels), zeros outside the image / past Cin."""
    n, h, w, cin = x.shape
    halo = np.zeros((chunks, HH * HW, 8))
    for c in range(chunks):
        for p in range(HH * HW):
            yy, xx = ty * TH - 1 + p // HW, tx * TW - 1 + p % HW
            if 0 <= yy < h and 0 <= xx < w:
                for e in range(8):
                    ch = c0 + 8 * c + e
                    halo[c, p, e] = x[batch, yy, xx, ch] if ch < cin else 0.0
    return halo


def read_operand(halo, start):
    """The 64 x 16 A operand a K-major no-swizzle descriptor (start, LBO, SBO) reads; byte offsets into the halo."""
    a = np.empty((64, 16))
    for r in range(64):
        for k in range(16):
            addr = start + (r // 8) * SBO + (r % 8) * 16 + (k // 8) * LBO + (k % 8) * 2
            chunk, within = divmod(addr, CHUNK)
            assert within < HH * HW * 16, "read past the 180 pixels of a chunk"
            a[r, k] = halo[chunk, within // 16, (within % 16) // 2]
    return a


def im2col(x, batch, ty, tx, mh, ky, kx, ch0):
    """Rows r of instruction mh = tile pixel (r / 8) * 16 + 8 * mh + r % 8; 16 channels from ch0."""
    n, h, w, cin = x.shape
    a = np.zeros((64, 16))
    for r in range(64):
        oy, ox = r // 8, 8 * mh + r % 8
        yy, xx = ty * TH + oy + ky - 1, tx * TW + ox + kx - 1
        if 0 <= yy < h and 0 <= xx < w:
            for k in range(16):
                if ch0 + k < cin:
                    a[r, k] = x[batch, yy, xx, ch0 + k]
    return a


@pytest.mark.parametrize("h,w,cin", [(16, 32, 128), (13, 21, 196), (9, 17, 256)])
def test_halo_descriptors_reproduce_im2col(h, w, cin):
    rs = np.random.RandomState(cin)
    x = rs.standard_normal((2, h, w, cin))
    cb = cin // 64 if cin % 64 <= 16 and cin > 64 else -(-cin // 64)
    rem = cin - 64 * cb
    tiles_h, tiles_w = -(-h // TH), -(-w // TW)
    for ty, tx in {(0, 0), (tiles_h - 1, tiles_w - 1), (0, tiles_w - 1)}:
        blocks = [(b, 8) for b in range(cb)] + ([(cb, 2)] if rem else [])
        for hh, chunks in blocks:
            halo = load_halo(x, 1, ty, tx, 64 * hh, chunks)
            for tap in range(9):
                ky, kx = divmod(tap, 3)
                for mh in range(2):
                    for kk in range(chunks // 2):
                        start = (ky * HW + 8 * mh + kx) * 16 + kk * 2 * LBO
                        got = read_operand(halo, start)
                        ref = im2col(x, 1, ty, tx, mh, ky, kx, 64 * hh + 16 * kk)
                        np.testing.assert_array_equal(got, ref)


def test_staging_rows_cover_the_tile_once():
    """Thread wt of a warpgroup holds rows r0 = 16 * (wt / 32) + (wt % 32) / 4 and r0 + 8 of each instruction; the
    kernel stages them at pixel rows p0 + 8 * mh and p0 + 8 * mh + 16, p0 = 32 * (wt / 32) + (wt % 32) / 4."""
    seen = {}
    for wt in range(128):
        r0 = 16 * (wt >> 5) + ((wt & 31) >> 2)
        p0 = 32 * (wt >> 5) + ((wt & 31) >> 2)
        for mh in range(2):
            for r, p in ((r0, p0 + 8 * mh), (r0 + 8, p0 + 8 * mh + 16)):
                assert p == (r // 8) * 16 + 8 * mh + r % 8
                seen[p] = seen.get(p, 0) + (wt & 3 == 0)
    assert sorted(seen) == list(range(128)) and set(seen.values()) == {1}
