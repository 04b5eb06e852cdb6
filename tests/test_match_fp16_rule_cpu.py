"""The accuracy rule of the fp16 transformer tests (tests/test_match_fp16_edges_gpu.py) against defects a kernel could
have.

One `self` and one `cross` encoder layer run, so a rounding flip of one layer cannot spread through later ones.  An
output of the fp16 kernels is held to

  max|kernel - emu64| <= 4 * max|emu32 - emu64| + 1e-6 * scale

where emu64 / emu32 are the float64 emulation of the fp16 semantics (tests/ref64.py, fp16=True) run in float64 and in
float32: the float32 run is the fp32 oracle of those semantics, as the fp32 numpy oracle is of the split mode's, and it
passes the rule by construction.  Each defect of ref64.DEFECTS, run in the float64 emulation in place of a kernel,
must fail the rule by at least 10x on both outputs; the defects that cannot are listed in BELOW_RULE with the cause and
fail that test (strict xfail)."""
import pytest
import torch

import loftr_b200.loftr as L
import ref64
import util
from test_kernel_edges_gpu import fp16_rule

F32 = torch.float32
# (n, L, S): L != S, partial 64-row tiles, S past two 64-key tiles; source keys [64, 128) masked, padding at the ends
SHAPES = [(1, 150, 200), (2, 97, 130), (1, 40, 140)]
# Token features: zero-mean (|x| up to about 10, the scale of the coarse transformer's), or with a common mode of 70 on
# every channel (|x| in [64, 128), where x - fp16(x) reaches 2^-5).  A defect is shown on the inputs where it is largest
# against the rounding noise of the float32 run.
INPUTS = {"zero_mean": (2.0, 1.0), "common_mode": (2.0, 70.0)}
# defect -> (inputs, attention kinds it applies to): Ksum exists in linear attention only, P's row sum in full only
DEFECTS = {"residual_hi": ("common_mode", ("linear", "full")), "p_row_sum": ("zero_mean", ("full",)),
           "ksum_exact": ("zero_mean", ("linear",)), "merge_block": ("zero_mean", ("linear", "full")),
           "key_tile": ("zero_mean", ("linear", "full"))}
# Defects the rule cannot see at 10x, with the measured cause (the factors over the bound are in DESIGN.md §16).  A
# float32 run differs from the float64 one in where fp16 roundings of the same value fall: each such flip moves one
# operand by an fp16 ulp, and after the LayerNorms the largest output moves by 1e-3 - 3e-3.  These defects perturb the
# attention by about 2^-12 / sqrt(keys) relative, averaged over the keys, which only re-draws those flips.
BELOW_RULE = {
    "p_row_sum": "P rounded in the row sum: 0.3x the bound, an averaged 2^-12 change under the fp32 rounding flips",
    "ksum_exact": "Ksum of the unrounded K: 0.2-0.3x the bound, an averaged 2^-12 change under the fp32 rounding flips",
}


def _layers(attention, seed=21):
    torch.manual_seed(seed)
    cfg = {"d_model": 256, "nhead": 8, "layer_names": ["self", "cross"], "attention": attention}
    return cfg, L.LocalFeatureTransformer(cfg, precision="fp16").eval()


def _inputs(n, l, s, kind, seed):
    amp, offset = INPUTS[kind]
    g = torch.Generator().manual_seed(seed)
    f0 = (torch.randn(n, l, 256, generator=g, dtype=torch.float64) * amp + offset).float()
    f1 = (torch.randn(n, s, 256, generator=g, dtype=torch.float64) * amp + offset).float()
    m0 = torch.ones(n, l, dtype=torch.bool)
    m1 = torch.ones(n, s, dtype=torch.bool)
    m0[:, l - 9:] = False
    m1[:, 64:128] = False
    m1[:, s - 5:] = False
    return f0, f1, m0, m1


def _emulate(tf, cfg, inp, dtype, defects=frozenset()):
    f0, f1, m0, m1 = inp
    old, ref64.DEFECTS = ref64.DEFECTS, frozenset(defects)
    try:
        return ref64.transformer(f0.to(dtype), f1.to(dtype), ref64.layer_weights(tf, dtype=dtype), cfg["layer_names"],
                                 8, m0, m1, cfg["attention"], fp16=True)
    finally:
        ref64.DEFECTS = old


CASES = [pytest.param(a, d, shape, id=f"{a}-{d}-n{shape[0]}_L{shape[1]}_S{shape[2]}",
                      marks=[pytest.mark.xfail(reason=BELOW_RULE[d], strict=True)] if d in BELOW_RULE else [])
         for a in ("linear", "full") for d, (_, kinds) in DEFECTS.items() if a in kinds for shape in SHAPES]


@pytest.mark.parametrize("attention,defect,shape", CASES)
def test_each_defect_fails_the_rule_by_10x(attention, defect, shape):
    """emu32 is within the rule by construction (and rounds somewhere: its error is not 0); the float64 emulation with
    the defect must exceed the rule's bound 10x on both outputs."""
    cfg, tf = _layers(attention)
    kind = DEFECTS[defect][0]
    inp = _inputs(*shape, kind, seed=sum(shape))
    emu64 = _emulate(tf, cfg, inp, torch.float64)
    emu32 = _emulate(tf, cfg, inp, F32)
    bad = _emulate(tf, cfg, inp, torch.float64, {defect})
    stats, factors = {"inputs": kind}, []
    for side in (0, 1):
        scale = emu64[side].abs().max().item()
        err32 = (emu32[side].double() - emu64[side]).abs().max().item()
        err = (bad[side] - emu64[side]).abs().max().item()
        assert 0 < err32 <= fp16_rule(err32, scale)
        factors.append(err / fp16_rule(err32, scale))
        stats.update({f"feat{side}_emu32_err": err32, f"feat{side}_defect_err": err, f"feat{side}_factor": factors[-1]})
    util.record(f"match_fp16_rule_{attention}_{defect}_n{shape[0]}_L{shape[1]}_S{shape[2]}", stats)
    assert min(factors) >= 10, f"{defect}: {factors[0]:.1f}x / {factors[1]:.1f}x the bound"


def test_the_emulation_keeps_its_dtype():
    """layer_weights gives float64 by default and exact float32 copies on request; a float32 run stays float32."""
    cfg, tf = _layers("full")
    inp = _inputs(1, 40, 140, "zero_mean", seed=3)
    w64, w32 = ref64.layer_weights(tf), ref64.layer_weights(tf, dtype=F32)
    assert all(v.dtype == torch.float64 for w in w64 for v in w.values())
    assert all(torch.equal(v.float(), w32[i][k]) for i, w in enumerate(w64) for k, v in w.items())
    assert all(o.dtype == F32 for o in _emulate(tf, cfg, inp, F32))
