"""gemm_split_kernel on single fp16 planes (EpiF16Operands, the kernels of match_precision "fp16") through lb_gemm_fp16,
at launches where every persistent CTA runs three or four output tiles, against a float64 product on the GPU.

Ring.  With one plane a ring stage holds 64 of K (twice the split mode's 32 in the same bytes), so a 128-row tile runs
K / 64 stages.  The ring has 4 stages at BLOCK_N = 256 (N > 128) and 6 at BLOCK_N = 128, and the fp32 accumulator is
staged over 3 of them at a tile's end: the three that end at the tile's last stage, or the ring's last three when those
would wrap (last stage 0 or 1).  Tile t of a CTA starts at ring stage t * stages % ring, so the launches below reach:

  BLOCK_N  ring  K     stages  last stage of tiles 0-3   staging wraps   next tile's first load is staged
  256      4     64    1       0 1 2 3                   tiles 0, 1      tiles 0, 1
  256      4     128   2       1 3 1 3                   tiles 0, 2      tiles 0, 2
  256      4     192   3       2 1 0 3                   tiles 1, 2      tiles 1, 2
  256      4     256   4       3 3 3 3                   never           never
  256      4     320   5       0 1 2 3                   tiles 0, 1      tiles 0, 1
  256      4     512   8       3 3 3 3                   never           never
  128      6     64    1       0 1 2 3                   tiles 0, 1      never
  128      6     128   2       1 3 5 1                   tiles 0, 3      never
  128      6     192   3       2 5 2 5                   never           never
  128      6     384   6       5 5 5 5                   never           never

K = 64 and 128 run 1 and 2 stages, fewer than the 3 the staging covers: the fine transformer's K = 128 products (q|k|v,
merge) are 2-stage tiles.  N = 96 runs one 128-wide column tile of which 96 columns are stored, N = 288 two 256-wide
ones of which the second stores 32 columns.  tests/test_pipeline_coverage_cpu.py replays this schedule from the ring
constants of the sources.

Bound.  The operands are fp16 values, so every product term is exact in fp32 and only the fp32 accumulation over K is
at fault: every element obeys

  |got - A B^T| <= K * 2^-23 * (|A| |B|^T)

with A B^T in float64.  A stale or skipped k-stage moves an element by about 1 / stages of (|A| |B|^T), far outside the
bound.  The lo pointers are passed as NULL: the kernel must not read them."""
import pytest
import torch

import util
from test_gemm_pipeline_gpu import block_n, launch_shape

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (N, K, batches, M % 128, per-batch B, A and B read as column slices of [rows, 2K] planes)
CASES = ([(256, k, 1, (1, 127)[i % 2], False, False) for i, k in enumerate((64, 128, 192, 256, 320, 512))]
         + [(96, k, 1, (127, 1)[i % 2], False, False) for i, k in enumerate((64, 128, 192, 384))]
         + [(288, 64, 1, 1, False, False), (288, 128, 1, 127, False, False)]
         + [(256, 192, 3, 1, False, False), (256, 128, 3, 1, True, False), (96, 128, 3, 1, True, False)]
         + [(256, 128, 1, 127, False, True), (256, 320, 3, 1, True, True), (96, 64, 1, 1, False, True)])


def _plane(x, wide):
    """fp16 [rows, K] -> itself, or the right half of a [rows, 2K] plane whose left half holds NaN."""
    if not wide:
        return x
    rows, k = x.shape
    p = torch.full((rows, 2 * k), float("nan"), dtype=torch.float16, device=DEV)
    p[:, k:] = x
    return p[:, k:]


def _gemm(a, b, out, batches, m, n, k, b_batched):
    """lb_gemm_fp16 on fp16 views a [batches * m, k] and b [(batches *) n, k] (no lo planes); out [batches * m, ldo]
    fp32."""
    from loftr_b200 import _lib
    from loftr_b200.loftr import _stream
    lda, ldb, ldo = a.stride(0), b.stride(0), out.stride(0)
    _lib.check(_lib.load().lb_gemm_fp16(a.data_ptr(), None, lda, m * lda, b.data_ptr(), None, ldb,
                                        n * ldb if b_batched else 0, out.data_ptr(), ldo, m * ldo, batches, m, n, k,
                                        _stream(out)))


@pytest.mark.parametrize("n,k,batches,rem,b_batched,wide", CASES)
def test_gemm_fp16_multi_tile_ctas_match_fp64(n, k, batches, rem, b_batched, wide):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m, m_tiles, items = launch_shape(n, batches, rem, sms)
    assert 3.5 * sms <= items <= 4 * sms and m % 128 == rem % 128
    g = torch.Generator(device=DEV).manual_seed(k * 1000 + n + batches + 7)
    a16 = (torch.randn(batches * m, k, device=DEV, generator=g) * 3 + 1).half()
    b16 = (torch.randn((batches if b_batched else 1) * n, k, device=DEV, generator=g) * 3 + 1).half()
    a, b = _plane(a16, wide), _plane(b16, wide)
    ldo = n + 32
    out = torch.full((batches * m, ldo), float("nan"), device=DEV)
    _gemm(a, b, out, batches, m, n, k, b_batched)
    again = torch.full_like(out, float("nan"))
    _gemm(a, b, again, batches, m, n, k, b_batched)

    a64 = a16.double().view(batches, m, k)
    b64 = b16.double().view(-1, n, k).expand(batches, n, k)
    ref = torch.bmm(a64, b64.transpose(1, 2))
    mag = torch.bmm(a64.abs(), b64.abs().transpose(1, 2))
    got = out[:, :n].double().view(batches, m, n)
    bound = k * 2.0 ** -23 * mag
    ratio = ((got - ref).abs() / bound).max().item()   # NaN (an unwritten element) fails the comparisons below
    rel = ((got - ref).abs().max() / ref.abs().max()).item()
    util.record(f"gemm_fp16_pipeline_N{n}_K{k}_b{batches}_r{rem}{'_bb' if b_batched else ''}{'_wide' if wide else ''}",
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
        _gemm(a[r0:], b, alone, 1, rows, n, k, False)
        assert torch.equal(alone[:, :n], out[r0:r0 + rows, :n]), f"m tile {mt} ({rows} rows) differs alone"
