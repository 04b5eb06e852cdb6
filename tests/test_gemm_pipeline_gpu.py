"""gemm_split_kernel (loftr_b200/csrc/gemm_split.cuh) through lb_gemm_split, at launches where every persistent CTA runs
three or four output tiles, against a float64 product on the GPU.

Ring.  With hi and lo planes a ring stage holds 32 of K, so a 128-row tile runs K / 32 stages.  The ring has 4 stages at
BLOCK_N = 256 (N > 128) and 6 at BLOCK_N = 128.  At a tile's end the fp32 accumulator is staged over 3 ring stages: the
three that end at the tile's last stage, or the ring's last three when those would wrap (last stage 0 or 1).  The next
tile's loads start after the last stage; the producer waits for the epilogue's release (acc_free) before it writes a
staged stage.  Tile t of a CTA starts at ring stage t * stages % ring, so the launches below reach:

  BLOCK_N  ring  K     stages  last stage of tiles 0-3   staging wraps   next tile's first load is staged
  256      4     64    2       1 3 1 3                   tiles 0, 2      tiles 0, 2
  256      4     128   4       3 3 3 3                   never           never
  256      4     192   6       1 3 1 3                   tiles 0, 2      tiles 0, 2
  256      4     256   8       3 3 3 3                   never           never
  256      4     320   10      1 3 1 3                   tiles 0, 2      tiles 0, 2
  256      4     1024  32      3 3 3 3                   never           never
  128      6     64    2       1 3 5 1                   tiles 0, 3      never
  128      6     128   4       3 1 5 3                   tile 1          never
  128      6     192   6       5 5 5 5                   never           never
  128      6     256   8       1 3 5 1                   tiles 0, 3      never
  128      6     384   12      5 5 5 5                   never           never

K = 64 runs 2 stages, fewer than the 3 the staging covers.  N = 96 runs one 128-wide column tile of which 96 columns
are stored, N = 288 two 256-wide ones of which the second stores 32 columns; N = 512 is two full ones.
tests/test_pipeline_coverage_cpu.py replays this schedule from the ring constants of the sources.

Bound.  The operands are split into fp16 planes, x = hi + lo + d with |d| <= 2^-22 |x| (while lo is a normal fp16
number), and each product is hi*hi + hi*lo + lo*hi: the two remainders and the dropped lo*lo term cost at most
3 * 2^-22 |a| |b| per term.  The fp32 accumulation over K adds at most K * 2^-23 of sum |a| |b|.  So every element obeys

  |got - ref| <= (3 * 2^-22 + K * 2^-23) * (|A| |B|^T)

A stale or skipped k-stage moves an element by about 1 / stages of (|A| |B|^T), far outside the bound.  The whole
matrix is also held to 5e-6 of its largest element, the bound of test_gemm_split_matches_fp64."""
import pytest
import torch

import util

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def block_n(n):
    """lb_gemm_split's column tile: 256 when N > 128, else 128."""
    return 256 if n > 128 else 128


# (N, K, batches, M % 128, per-batch B, A and B read as column slices of [rows, 2K] planes)
CASES = ([(256, k, 1, (1, 127)[i % 2], False, False) for i, k in enumerate((64, 128, 192, 256, 320, 1024))]
         + [(96, k, 1, (127, 1)[i % 2], False, False) for i, k in enumerate((64, 128, 192, 256, 384))]
         + [(288, 64, 1, 1, False, False), (512, 64, 1, 127, False, False)]
         + [(256, 192, 3, 1, False, False), (256, 192, 3, 1, True, False), (96, 256, 3, 1, True, False)]
         + [(256, 256, 1, 127, False, True), (256, 320, 3, 1, True, True)])


def launch_shape(n, batches, rem, sms):
    """(M, m_tiles, items): the fewest 128-row tiles per batch that give at least 3.5 x SMs work items, the last tile
    holding `rem` rows."""
    n_tiles = -(-n // block_n(n))
    m_tiles = -(-(7 * sms) // (2 * batches * n_tiles))
    return (m_tiles - 1) * 128 + rem, m_tiles, batches * m_tiles * n_tiles


def _planes(x, wide):
    """fp32 [rows, K] -> fp16 (hi, lo) views with row stride K, or the right halves of [rows, 2K] planes whose left
    halves hold NaN."""
    from loftr_b200.loftr import split_planes
    if not wide:
        return split_planes(x)
    rows, k = x.shape
    hi = torch.full((rows, 2 * k), float("nan"), dtype=torch.float16, device=DEV)
    lo = torch.full((rows, 2 * k), float("nan"), dtype=torch.float16, device=DEV)
    split_planes(x, hi, lo, col0=k)
    return hi[:, k:], lo[:, k:]


def _gemm(a, b, out, batches, m, n, k, b_batched):
    """lb_gemm_split on plane views a = (hi, lo) [batches * m, k] and b = (hi, lo) [(batches *) n, k]; out
    [batches * m, ldo] fp32."""
    from loftr_b200 import _lib
    from loftr_b200.loftr import _stream
    lda, ldb, ldo = a[0].stride(0), b[0].stride(0), out.stride(0)
    _lib.check(_lib.load().lb_gemm_split(a[0].data_ptr(), a[1].data_ptr(), lda, m * lda, b[0].data_ptr(),
                                         b[1].data_ptr(), ldb, n * ldb if b_batched else 0, out.data_ptr(), ldo,
                                         m * ldo, batches, m, n, k, _stream(out)))


@pytest.mark.parametrize("n,k,batches,rem,b_batched,wide", CASES)
def test_gemm_split_multi_tile_ctas_match_fp64(n, k, batches, rem, b_batched, wide):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m, m_tiles, items = launch_shape(n, batches, rem, sms)
    assert 3.5 * sms <= items <= 4 * sms and m % 128 == rem % 128
    g = torch.Generator(device=DEV).manual_seed(k * 1000 + n + batches)
    a32 = torch.randn(batches * m, k, device=DEV, generator=g) * 3 + 1
    b32 = torch.randn((batches if b_batched else 1) * n, k, device=DEV, generator=g) * 3 + 1
    a, b = _planes(a32, wide), _planes(b32, wide)
    ldo = n + 32
    out = torch.full((batches * m, ldo), float("nan"), device=DEV)
    _gemm(a, b, out, batches, m, n, k, b_batched)
    again = torch.full_like(out, float("nan"))
    _gemm(a, b, again, batches, m, n, k, b_batched)

    a64 = a32.double().view(batches, m, k)
    b64 = b32.double().view(-1, n, k).expand(batches, n, k)
    ref = torch.bmm(a64, b64.transpose(1, 2))
    mag = torch.bmm(a64.abs(), b64.abs().transpose(1, 2))
    got = out[:, :n].double().view(batches, m, n)
    bound = (3 * 2.0 ** -22 + k * 2.0 ** -23) * mag
    ratio = ((got - ref).abs() / bound).max().item()   # NaN (an unwritten element) fails the comparisons below
    rel = ((got - ref).abs().max() / ref.abs().max()).item()
    util.record(f"gemm_pipeline_N{n}_K{k}_b{batches}_r{rem}{'_bb' if b_batched else ''}{'_wide' if wide else ''}",
                {"sms": sms, "items": items, "worst_err_over_bound": ratio, "max_err_over_max_ref": rel})
    assert ratio <= 1.0, f"an element exceeds the bound by {ratio:.3f}x"
    assert rel < 5e-6, f"max error {rel:.3e} of the largest element"
    assert torch.isnan(out[:, n:]).all(), "columns past N were written"
    assert torch.equal(out[:, :n], again[:, :n]), "two identical launches differ"

    if batches > 1:
        return
    # a 128-row tile gives the same bits launched alone (stage 0 of CTA 0) as inside the big launch, where items
    # [2 grid, 3 grid) are a CTA's third tile and [3 grid, items) its fourth; the last one is the ragged tile
    n_tiles = items // m_tiles
    grid = sms
    for mt in sorted({2 * grid // n_tiles, (3 * grid + 5) // n_tiles, m_tiles - 1}):
        assert mt * n_tiles >= 2 * grid
        r0 = mt * 128
        rows = min(128, m - r0)
        alone = torch.full((rows, ldo), float("nan"), device=DEV)
        _gemm((a[0][r0:], a[1][r0:]), b, alone, 1, rows, n, k, False)
        assert torch.equal(alone[:, :n], out[r0:r0 + rows, :n]), f"m tile {mt} ({rows} rows) differs alone"
