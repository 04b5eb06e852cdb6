"""What tests/test_gemm_pipeline_gpu.py, tests/test_gemm_pipeline_fp16_gpu.py and tests/test_backbone_widths_gpu.py
reach, replayed on the CPU from the ring constants of the sources (read with regular expressions) and a mirror of
engine.cu's conv_layout.  These tests fail when a change to the kernels' shared-memory budget or to those files' cases
leaves the tile hand-off or the convolution layouts they were written for uncovered."""
import collections
import os
import re

import pytest
import torch

import test_backbone_widths_gpu as widths
import test_gemm_pipeline_fp16_gpu as pipeline16
import test_gemm_pipeline_gpu as pipeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "loftr_b200", "csrc")
SRC = {f: open(os.path.join(CSRC, f)).read() for f in ("gemm_split.cuh", "conv_halo.cuh", "epilogues.cuh", "engine.cu")}


def _int(pattern, f):
    """The integer expression (digits, * and +) that `pattern`'s group 1 captures in source file f."""
    m = re.search(pattern, SRC[f])
    assert m, f"{pattern} not found in {f}"
    assert re.fullmatch(r"[\d\s*+()]+", m.group(1)), m.group(1)
    return eval(m.group(1))


BLOCK_M = _int(r"constexpr int kBlockM = ([^;]+);", "gemm_split.cuh")
BLOCK_K = _int(r"constexpr int kBlockK = ([^;]+);", "gemm_split.cuh")
REM_CHANNELS = _int(r"constexpr int kRemChannels = ([^;]+);", "gemm_split.cuh")
SMEM_LIMIT = _int(r"constexpr int kSmemLimit = ([^;]+);", "gemm_split.cuh")
BAR_BYTES = _int(r"kBarBytes = ([^;]+);", "gemm_split.cuh")
RING_WANT = _int(r"kWant = ([^/]+) / kStageBytes;", "gemm_split.cuh")
ACC_PAD = _int(r"acc_stride\(int block_n\) \{ return block_n \+ ([^;]+); \}", "gemm_split.cuh")
ACC_TAIL = _int(r"acc_bytes\(int block_n\) \{ return \(kBlockM \* acc_stride\(block_n\) \+ ([^)]+)\) \* 4; \}",
                "gemm_split.cuh")
HALO_CHUNK = _int(r"constexpr int kHaloChunkBytes = ([^;]+);", "conv_halo.cuh")
HALO_BAR_BYTES = _int(r"kBarBytes = ([^;]+);", "conv_halo.cuh")
HALO_MAX_STAGES = _int(r"kStages = kFree / kStageBytes < (\d+) \?", "conv_halo.cuh")
EPI_SCRATCH = _int(r"constexpr int kEpiScratchBytes = ([^;]+);", "epilogues.cuh")
OWN_XPOSE = _int(r"kSmemBytes = kXposeOffset \+ \(kOwnXpose \? ([^:]+) :", "epilogues.cuh")
TAPS = 9


def gemm_ring(bn, epi_bytes, planes=2):
    """GemmSmem<bn, epi_bytes, planes> (hi and lo planes, or hi only): (K per stage, ring stages, stages under the
    staged accumulator, remainder taps per stage)."""
    bk = BLOCK_K // planes
    stage = planes * (BLOCK_M + bn) * bk * 2
    stages = min((SMEM_LIMIT - BAR_BYTES - epi_bytes) // stage, RING_WANT // stage)
    acc_stages = -(-((BLOCK_M * (bn + ACC_PAD) + ACC_TAIL) * 4) // stage)
    assert acc_stages < stages
    return bk, stages, acc_stages, stage // (planes * (BLOCK_M + bn) * REM_CHANNELS * 2)


def conv_epi_bytes(bn, upsample):
    """EpiConvImpl<bn, upsample, .>::kSmemBytes"""
    return EPI_SCRATCH + 2 * (-(-bn // 32) * 32) * 4 + (OWN_XPOSE if bn == 208 and not upsample else 0)


def halo_subs(bn):
    """Weight stages per (tap, 64-channel block) of conv3x3_halo_kernel<bn> with hi and lo planes (HaloSmem: kBlockK /
    kBK)."""
    free = SMEM_LIMIT - HALO_BAR_BYTES - conv_epi_bytes(bn, False) - 2 * 2 * (BLOCK_K // 8) * HALO_CHUNK
    bk = BLOCK_K if free // (2 * bn * BLOCK_K * 2) >= 3 else BLOCK_K // 2
    assert min(free // (2 * bn * bk * 2), HALO_MAX_STAGES) >= 3
    return BLOCK_K // bk


def conv_layout(cin):
    """engine.cu conv_layout: (64-channel blocks per tap, remainder channels per tap)."""
    r = cin % BLOCK_K
    if cin > BLOCK_K and 0 < r <= REM_CHANNELS:
        return cin // BLOCK_K, r
    return -(-cin // BLOCK_K), 0


def test_conv_layout_mirror_matches_the_library():
    import ctypes as C
    from loftr_b200 import _lib
    lib = _lib.load()
    for cin in range(1, 257):
        cb, rem = C.c_int(), C.c_int()
        _lib.check(lib.lb_conv_layout(cin, C.byref(cb), C.byref(rem)))
        assert (cb.value, rem.value) == conv_layout(cin), cin


def gemm_schedule(n, k, batches, rem, sms, planes=2):
    """Per CTA of one lb_gemm_split (planes = 2) or lb_gemm_fp16 (planes = 1) launch: a list of (last ring stage,
    staging wraps, next tile's first load lands in a staged stage) for each of its tiles."""
    bk, ring, acc, _ = gemm_ring(pipeline.block_n(n), EPI_SCRATCH, planes)
    _, _, items = pipeline.launch_shape(n, batches, rem, sms)
    grid = min(items, sms)
    stages = k // bk
    ctas = []
    for cta in range(grid):
        pos, tiles = 0, []
        for _ in range(cta, items, grid):
            last = (pos + stages - 1) % ring
            first = last - acc + 1 if last >= acc - 1 else ring - acc
            tiles.append((last, last < acc - 1, first <= (last + 1) % ring < first + acc))
            pos = (pos + stages) % ring
        ctas.append(tiles)
    return ctas


def test_gemm_rings_are_the_ones_the_tables_describe():
    """lb_gemm_split's and lb_gemm_fp16's epilogue (EpiActStore, with EpiF16Operands adding nothing but the plane
    count) takes kEpiScratchBytes, and its rings are those of the tables in tests/test_gemm_pipeline_gpu.py and
    tests/test_gemm_pipeline_fp16_gpu.py: 32 / 64 of K per stage with two planes / one, 4 / 6 stages at BLOCK_N
    256 / 128, 3 under the staging."""
    m = re.search(r"struct EpiActStore \{.*?kSmemBytes = (\w+);", SRC["epilogues.cuh"], re.S)
    assert m and m.group(1) == "kEpiScratchBytes"
    m = re.search(r"struct EpiF16Operands : Epi \{(.*?)\};", SRC["epilogues.cuh"], re.S)
    assert m and m.group(1).split() == ["using", "Epi::Epi;", "static", "constexpr", "int", "kOperandPlanes", "=", "1;"]
    m = re.search(r"static int gemm_test\(.*?\n\}\n", SRC["engine.cu"], re.S)
    assert m, "gemm_test not found in engine.cu"
    assert re.findall(r"using Epi = Operands<EpiActStore<(\d+)>, kP>;", m.group(0)) == ["256", "128"]
    assert re.search(r"int lb_gemm_split\([^{]*\{\s*return gemm_test<2>\(", SRC["engine.cu"])
    assert re.search(r"int lb_gemm_fp16\([^{]*\{\s*return gemm_test<1>\(", SRC["engine.cu"])
    assert [gemm_ring(bn, EPI_SCRATCH)[:3] for bn in (256, 128)] == [(32, 4, 3), (32, 6, 3)]
    assert [gemm_ring(bn, EPI_SCRATCH, 1)[:3] for bn in (256, 128)] == [(64, 4, 3), (64, 6, 3)]


@pytest.mark.parametrize("sms", [114, 132])
def test_gemm_pipeline_launches_reach_the_tile_hand_off(sms):
    wraps, no_wraps, staged_first_load, k64 = 0, 0, 0, False
    for n, k, batches, rem, _, _ in pipeline.CASES:
        ctas = gemm_schedule(n, k, batches, rem, sms)
        counts = {len(t) for t in ctas}
        assert len(ctas) == sms and counts == {3, 4}, (n, k, batches, counts)
        tiles = [t for c in ctas for t in c]
        wraps += sum(w for _, w, _ in tiles)
        no_wraps += sum(not w for _, w, _ in tiles)
        staged_first_load += sum(s for c in ctas for _, _, s in c[:-1])   # a next tile on the same CTA
        k64 |= k == 64
    assert wraps and no_wraps and staged_first_load and k64
    assert {pipeline.block_n(n) for n, *_ in pipeline.CASES} == {128, 256}


@pytest.mark.parametrize("sms", [114, 132])
def test_gemm_fp16_pipeline_launches_reach_the_tile_hand_off(sms):
    """The one-plane ring at both column tiles: staging that wraps and that does not, 1- and 2-stage tiles (fewer than
    the 3 the staging covers), and at BLOCK_N 256 a next tile whose first load lands in the staging.  At BLOCK_N 128
    (ring 6, staging 3) no ring position can stage the next tile's first load."""
    seen = {bn: collections.Counter() for bn in (128, 256)}
    for n, k, batches, rem, _, _ in pipeline16.CASES:
        ctas = gemm_schedule(n, k, batches, rem, sms, planes=1)
        counts = {len(t) for t in ctas}
        assert len(ctas) == sms and counts == {3, 4}, (n, k, batches, counts)
        c = seen[pipeline.block_n(n)]
        tiles = [t for cta in ctas for t in cta]
        c["wrap"] += sum(w for _, w, _ in tiles)
        c["no_wrap"] += sum(not w for _, w, _ in tiles)
        c["staged_first_load"] += sum(s for cta in ctas for _, _, s in cta[:-1])
        c[f"stages_{k // BLOCK_K}"] += 1
    for bn, c in seen.items():
        assert c["wrap"] and c["no_wrap"] and c["stages_1"] and c["stages_2"], (bn, c)
    assert seen[256]["staged_first_load"]
    _, ring, acc, _ = gemm_ring(128, EPI_SCRATCH, 1)
    for last in range(ring):
        first = last - acc + 1 if last >= acc - 1 else ring - acc
        assert not first <= (last + 1) % ring < first + acc
    assert {k for n, k, *_ in pipeline16.CASES if pipeline.block_n(n) == 256} == {64, 128, 192, 256, 320, 512}
    assert {k for n, k, *_ in pipeline16.CASES if pipeline.block_n(n) == 128} == {64, 128, 192, 384}


Conv = collections.namedtuple("Conv", "kind cin cout cin_blocks rem halos tap_major bn stages ring")


def conv_table(d2, d3):
    """A Conv per convolution after the stem of ResNetFPN(128, [128, d2, d3]) on the split-precision path: halo kernel
    or gemm_split_kernel, channel layout, output tile, k-stages per tile and (gemm mode) ring stages."""
    from loftr_b200.backbone import ResNetFPN
    with torch.device("meta"):
        m = ResNetFPN(128, [128, d2, d3])
    rows = []
    for name, c in m.named_modules():
        if not isinstance(c, torch.nn.Conv2d) or name == "conv1":
            continue
        cin, cout, k, stride = c.in_channels, c.out_channels, c.kernel_size[0], c.stride[0]
        up = name in ("layer1_outconv", "layer2_outconv")   # the FPN laterals carry the upsample-add
        cb, rem = conv_layout(cin)
        if k == 3 and stride == 1 and not up:
            bn = 128 if cout <= 128 else 200 if cout <= 200 else 256
            halos = cb + (rem > 0)
            rows.append(Conv("halo", cin, cout, cb, rem, halos, halos <= 2, bn,
                             TAPS * (cb * halo_subs(bn) + (rem > 0)), None))
        else:
            bn = 128 if cout <= 128 else 208 if cout <= 208 else 256
            bk, ring, _, rem_taps = gemm_ring(bn, conv_epi_bytes(bn, up))
            stages = k * k * cb * (BLOCK_K // bk) + (-(-k * k // rem_taps) if rem else 0)
            rows.append(Conv("gemm", cin, cout, cb, rem, None, None, bn, stages, ring))
    return rows


def test_backbone_widths_reach_every_convolution_layout():
    rows = [r for d2, d3 in widths.WIDTHS for r in conv_table(d2, d3)]
    halo = [r for r in rows if r.kind == "halo"]
    assert {40, 64, 72, 80, 81, 136, 160, 193, 208, 209, 256} <= {r.cin for r in halo}
    assert {r.halos for r in halo} == {1, 2, 3, 4}
    assert any(r.tap_major and r.rem for r in halo), "tap-major order with a remainder halo"
    assert any(not r.tap_major for r in halo), "channel-block-major order"
    assert any(r.cin < BLOCK_K for r in halo), "one zero-padded channel block"
    assert {1, 8, REM_CHANNELS} <= {r.rem for r in halo}
    assert any(r.cin % BLOCK_K == REM_CHANNELS + 1 and r.cin_blocks == 4 for r in halo), "r = 17: a padded 4th block"
    couts = lambda kind, bn: {r.cout for r in rows if r.kind == kind and r.bn == bn}
    assert min(couts("halo", 128)) < 128 and 128 in couts("halo", 128)
    assert any(128 < c < 196 for c in couts("halo", 200)) and any(196 < c <= 200 for c in couts("halo", 200))
    assert any(200 < c < 256 for c in couts("halo", 256)) and 256 in couts("halo", 256)
    assert any(128 < c < 208 for c in couts("gemm", 208)) and 208 in couts("gemm", 208)
    assert any(208 < c < 256 for c in couts("gemm", 256))
    assert {40, 64, 72, 80, 136, 160, 200, 208} <= {d3 for _, d3 in widths.WIDTHS}
    for bn in (208, 256):
        assert any(r.kind == "gemm" and r.bn == bn and r.stages % r.ring for r in rows), \
            f"no gemm-mode layer at BN {bn} ends a tile mid-ring"
