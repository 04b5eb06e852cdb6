"""Float64 references of the tensor-core backbone (lb_backbone_forward / lb_backbone_forward_fp16), per stage and end
to end, and the helpers of the backbone tests.

The backbone keeps every activation in its workspace (NHWC fp16 planes, carved by `carve_bb` in
loftr_b200/csrc/engine.cu).  `workspace_layout` mirrors that carve, so a test can read each convolution's stored
inputs and output after one forward and judge every stage on its own: the reference of a stage starts from what the
kernels stored, never from upstream float64 values, so errors do not compound and a failure names its layer.

`STAGES` lists the stages in launch order.  A stage is one convolution, or a chain of two where the first one's
output buffer is overwritten later in the forward (t1, t2, t3).  `run_stage` evaluates a stage in float64 or float32
with the fp32 weights (the split path's reference and oracle) or with the fp16 weights fp16(w * 2^e) * 2^-e of the
fp16 path, BatchNorm folded.  `STAGES` is the only description of the network in the tests: `forward_f64` runs it end
to end.

`forward_f64(m, images, fp16=True)` is the float64 emulation of the fp16 backbone (`backbone_impl="b200_fp16"`;
DESIGN.md §15).  Every convolution after the stem multiplies the stored fp16 activation by fp16(w * 2^e) (e =
`weight_exponent` of the layer's weights, the exponent of the split path) and accumulates exactly; the epilogue applies
the folded BatchNorm, the residual, the FPN x2 bilinear upsample-add (align_corners=True) and the activation, in that
order, and the result is stored as one fp16 plane (round to nearest even).  Residual and upsample addends are the
stored fp16 values.  The stem's product stays split (within fp32 of exact here) and only its output is rounded.
feat_c and feat_f are the epilogue values before rounding (the kernels write them in fp32).  With fp16=False nothing
is rounded and the weights are fp32: the float64 ResNetFPN_8_2 forward, which pins STAGES' fold, residual, upsample
and activation structure.

`split_stage` is the float64 emulation of the split path's semantics (DESIGN.md §2): fp16 hi / lo planes of the
activation and of w * 2^e, the products hi*hi + hi*lo + lo*hi accumulated exactly, the epilogue's value rounded to
fp32 and stored as hi + lo planes.  Its `defect` argument removes one part of those semantics, which is how
tests/test_backbone_stages_cpu.py shows that the stage rule catches such bugs."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.nn.functional as F

from ref64 import r16

# The grid of tests/test_backbone_stages_gpu.py: (N, H, W) and (d2, d3) of ResNetFPN(128, [128, d2, d3])
GRID_SHAPES = [(1, 8, 8), (1, 16, 16), (3, 72, 88), (1, 8, 1024), (1, 512, 8), (8, 136, 200), (1, 480, 640)]
GRID_WIDTHS = [(196, 256), (81, 208), (193, 80), (40, 160)]


def make_backbone(d2, d3, device):
    """ResNetFPN(128, [128, d2, d3]) in eval mode with the weights and BatchNorm statistics of tests/golden/weights.py"""
    import weights as W
    from loftr_b200.backbone import ResNetFPN
    m = ResNetFPN(128, [128, d2, d3]).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    m.load_state_dict({k: torch.from_numpy(v) for k, v in W.make_state(shapes, seed=d2 * 1000 + d3).items()})
    return m.to(device)


def image(shape, seed, device="cuda:0"):
    """(N, H, W) -> a uniform [0, 1) float32 batch [N, 1, H, W] on `device`"""
    n, h, w = shape
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.uniform(0, 1, (n, 1, h, w)).astype(np.float32)).to(device)


def backbone_forward(tc, img, fill=0):
    """TensorCoreBackbone.__call__ (lb_backbone_forward, or lb_backbone_forward_fp16 for precision "fp16") into a
    workspace of our own pre-filled with byte `fill` (0xFF: every fp16 is NaN) -> (workspace bytes, feat_c, feat_f),
    the feature maps fp32 NHWC as the kernels wrote them."""
    from loftr_b200 import _lib
    from loftr_b200.loftr import _stream
    lib = _lib.load()
    w, _ = tc._pack()
    n, _, h, wd = img.shape
    fp16 = tc.precision == "fp16"
    workspace_bytes = lib.lb_backbone_workspace_bytes_fp16 if fp16 else lib.lb_backbone_workspace_bytes
    forward = lib.lb_backbone_forward_fp16 if fp16 else lib.lb_backbone_forward
    feat_c = torch.empty(n, h // 8, wd // 8, tc.m.layer3_outconv.out_channels, dtype=torch.float32, device=img.device)
    feat_f = torch.empty(n, h // 2, wd // 2, 128, dtype=torch.float32, device=img.device)
    ws = torch.full((workspace_bytes(C.byref(w), n, h, wd),), fill, dtype=torch.uint8, device=img.device)
    _lib.check(forward(C.byref(w), img.data_ptr(), n, h, wd, feat_c.data_ptr(), feat_f.data_ptr(), ws.data_ptr(),
                       ws.numel(), _stream(img)))
    torch.cuda.synchronize()
    return ws, feat_c, feat_f


# ------------------------------------------------------------------------------------------------ workspace mirror
# carve_bb (loftr_b200/csrc/engine.cu): (name, resolution divisor, width index into (d1, d2, d3)) in carve order
BUFFERS = [("s0", 2, 0), ("t1", 2, 0), ("a1", 2, 0), ("x1", 2, 0),
           ("t2", 4, 1), ("dn2", 4, 1), ("a2", 4, 1), ("x2", 4, 1),
           ("t3", 8, 2), ("dn3", 8, 2), ("a3", 8, 2), ("x3", 8, 2), ("x3o", 8, 2),
           ("x2l", 4, 2), ("m2", 4, 2), ("x2o", 4, 1),
           ("x1l", 2, 1), ("m1", 2, 1)]


def _take(off, nbytes):
    """Bump::take: every allocation is rounded up to 256 bytes"""
    return off + ((nbytes + 255) & ~255)


def workspace_layout(n, h, w, dims, planes):
    """carve_bb for an N x H x W batch and widths dims = (d1, d2, d3) with `planes` fp16 planes (2: split, 1: fp16) ->
    ({name: (hi byte offset, lo byte offset or None, (n, h, w, channels), row stride)}, total bytes).  The library
    sizes its workspace as total + 256."""
    out, off = {}, 0
    for name, div, k in BUFFERS:
        c = dims[k]
        ld = (c + 7) & ~7
        nbytes = n * (h // div) * (w // div) * ld * 2
        hi = off
        off = _take(off, nbytes)
        lo = None
        if planes == 2:
            lo = off
            off = _take(off, nbytes)
        out[name] = (hi, lo, (n, h // div, w // div, c), ld)
    return out, off


def decode(ws, entry):
    """One workspace buffer -> float64 NCHW (hi + lo, or hi), channels [0, C) only"""
    hi_off, lo_off, (n, h, w, c), ld = entry
    count = n * h * w * ld

    def plane(off):
        return ws[off:off + 2 * count].view(torch.float16).view(n, h, w, ld)[..., :c].double()
    x = plane(hi_off) if lo_off is None else plane(hi_off) + plane(lo_off)
    return x.permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ stages
# A step: (module path of the conv, module path of its BatchNorm or None, activation, input, residual, upsample source,
# output).  Outputs starting with "_" are overwritten later in the forward: they stay inside their stage.
def _unit(layer, i, inp, skip, mid, out):
    p = f"layer{layer}.{i}"
    return [(f"{p}.conv1", f"{p}.bn1", "relu", inp, None, None, mid), (f"{p}.conv2", f"{p}.bn2", "relu", mid, skip, None, out)]


def _layer_stages(lv, inp):
    t, dn, a, x = f"t{lv}", f"dn{lv}", f"a{lv}", f"x{lv}"
    c = f"layer{lv}.0.downsample"
    return [(f"l{lv}.down", "gemm", [(f"{c}.0", f"{c}.1", None, inp, None, None, dn)]),
            (f"l{lv}.0-1", "gemm+halo", _unit(lv, 0, inp, dn, "_" + t, a)),
            (f"l{lv}.2", "halo", _unit(lv, 1, a, a, t, x)[:1]),
            (f"l{lv}.3", "halo", [(f"layer{lv}.1.conv2", f"layer{lv}.1.bn2", "relu", t, a, None, x)])]


# (stage name, kernel class, steps); the stem's single step has the image as input
STAGES = ([("stem", "stem", [("conv1", "bn1", "relu", "image", None, None, "s0")]),
           ("l1.0-1", "halo", _unit(1, 0, "s0", "s0", "_t1", "a1")),
           ("l1.2", "halo", _unit(1, 1, "a1", "a1", "t1", "x1")[:1]),
           ("l1.3", "halo", [("layer1.1.conv2", "layer1.1.bn2", "relu", "t1", "a1", None, "x1")])]
          + _layer_stages(2, "x1") + _layer_stages(3, "x2")
          + [("l3_out", "gemm", [("layer3_outconv", None, None, "x3", None, None, "x3o")]),
             ("l2_out", "upsample", [("layer2_outconv", None, None, "x2", None, "x3o", "x2l")]),
             ("l2_out2.0", "halo", [("layer2_outconv2.0", "layer2_outconv2.1", "leaky", "x2l", None, None, "m2")]),
             ("l2_out2.1", "halo", [("layer2_outconv2.3", None, None, "m2", None, None, "x2o")]),
             ("l1_out", "upsample", [("layer1_outconv", None, None, "x1", None, "x2o", "x1l")]),
             ("l1_out2.0", "halo", [("layer1_outconv2.0", "layer1_outconv2.1", "leaky", "x1l", None, None, "m1")]),
             ("l1_out2.1", "halo", [("layer1_outconv2.3", None, None, "m1", None, None, "feat_f")])])
# the fp32 feature maps: feat_c is written beside x3o by the same epilogue, feat_f is the last convolution's output
FP32_OUTPUTS = {"x3o": "feat_c", "feat_f": "feat_f"}


def _weight(conv, weights, dtype):
    from loftr_b200.loftr import weight_exponent
    w = conv.weight.detach().float()
    if weights == "fp16":
        e = weight_exponent(w)
        return (w * 2.0 ** e).half().to(dtype) * 2.0 ** (-e)
    return w.to(dtype)


def _bn(bn, dtype):
    """Folded BatchNorm -> (scale, shift) in `dtype` (float32: like TensorCoreBackbone._fold)"""
    scale = bn.weight.detach().to(dtype) / torch.sqrt(bn.running_var.detach().to(dtype) + bn.eps)
    return scale, bn.bias.detach().to(dtype) - bn.running_mean.detach().to(dtype) * scale


def conv_step(m, step, get, dtype, weights="fp32"):
    """One convolution with its epilogue: act(bn(conv(x)) + residual + up_x2(source)) in `dtype`.  `get(name)` returns
    a stored buffer (NCHW, any float dtype).  The stem always uses the fp32 weights: its product stays split in both
    precisions."""
    conv_p, bn_p, act, inp, res, up, _ = step
    conv = m.get_submodule(conv_p)
    wt = _weight(conv, "fp32" if conv_p == "conv1" else weights, dtype)
    y = F.conv2d(get(inp).to(dtype), wt, stride=conv.stride, padding=conv.padding)
    if bn_p is not None:
        scale, shift = _bn(m.get_submodule(bn_p), dtype)
        y = y * scale.to(y.device).view(1, -1, 1, 1) + shift.to(y.device).view(1, -1, 1, 1)
    if res is not None:
        y = y + get(res).to(dtype)
    if up is not None:
        y = y + F.interpolate(get(up).to(dtype), scale_factor=2.0, mode="bilinear", align_corners=True)
    if act == "relu":
        y = F.relu(y)
    elif act == "leaky":
        y = F.leaky_relu(y, 0.01)
    return y


def run_stage(m, steps, get, dtype, weights="fp32", store=None):
    """Evaluate a stage from stored inputs -> its final output (unrounded).  `store` rounds a chain's intermediate the
    way the kernel stored it (fp16 for the fp16 path); without it the chain stays in `dtype`."""
    mid = {}
    look = lambda name: mid[name] if name in mid else get(name)
    y = None
    for step in steps:
        y = conv_step(m, step, look, dtype, weights)
        mid[step[6]] = store(y) if store is not None else y
    return y


def forward_f64(m, images, fp16=True):
    """STAGES end to end in float64: the fp16 path's emulation (fp16 weights, every stored activation rounded to fp16)
    or, with fp16=False, the exact forward.  m: the PyTorch ResNetFPN; images [N, 1, H, W] -> (feat_c, feat_f)
    float64 NCHW, on the device of `images` (m must live there too)."""
    store = r16 if fp16 else None
    bufs, feats = {"image": images.detach().double()}, {}
    for _, _, steps in STAGES:
        out = steps[-1][6]
        y = run_stage(m, steps, bufs.__getitem__, torch.float64, "fp16" if fp16 else "fp32", store)
        bufs[out] = store(y) if fp16 else y
        if out in FP32_OUTPUTS:
            feats[FP32_OUTPUTS[out]] = y
    return feats["feat_c"], feats["feat_f"]


# Finding, measured on an H100 80GB HBM3 at 700 W: the 3x3 stages (conv3x3_halo_kernel, and the strided 3x3 of
# gemm_split_kernel inside the chains) exceed 4x the fp32 oracle's error -- up to 11.6x on the split path and 4.8x on
# feat_f of the fp16 path -- while the stem and the 1x1 convolutions (K <= 256) stay within it.  The excess grows with
# the number of wgmma accumulation steps (9 taps x Cin / 16 per plane, three planes on the split path) and the errors
# shrink |ref| (recorded `bias` near -1 on the linear outputs): the tensor cores' fp32 accumulation truncates, where
# the oracle's fp32 FMA chain rounds to nearest.  The float64 emulation with exact accumulation stays at 0.1x of the
# bound (tests/test_backbone_stages_cpu.py).  These stages are held to 16x the oracle's error and, on the fp16 path, to
# 2 % of stored values off fp16(ref); every defect of the CPU test still exceeds that.
FINDING_STAGES = {name for name, cls, _ in STAGES if "halo" in cls}
FINDING_FACTOR = 16
FINDING_SHARE = 0.02


# ------------------------------------------------------------------------------------------------ split emulation
DEFECTS = ("hi_lo_dropped", "lo_hi_dropped", "lo_plane_not_stored", "remainder_hi_only")
BLOCK_K, REM_CHANNELS = 64, 16


def conv_layout(cin):
    """lb_conv_layout: (channel blocks of 64, remainder channels kept in their own 16-wide planes)"""
    r = cin % BLOCK_K
    if cin > BLOCK_K and 0 < r <= REM_CHANNELS:
        return cin // BLOCK_K, r
    return -(-cin // BLOCK_K), 0


def split_planes(x):
    """split_f16 of fp32 values: hi = fp16(x), lo = fp16(x - hi), returned as float64"""
    x = x.float()
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi.double(), lo.double()


def store_split(y, defect=None):
    """The epilogue value (float64) -> fp32 -> the stored hi + lo planes (hi only under `lo_plane_not_stored`)"""
    hi, lo = split_planes(y)
    return hi if defect == "lo_plane_not_stored" else hi + lo


def split_stage(m, steps, get, defect=None):
    """Float64 emulation of the split path for a stage (stored hi + lo inputs from `get`): exact accumulation of
    hi*hi + hi*lo + lo*hi (activation x weight), epilogue in float64, output stored through `store_split`.  A chain's
    intermediate is stored the same way."""
    from loftr_b200.loftr import weight_exponent
    mid = {}
    look = lambda name: mid[name] if name in mid else get(name)
    y = None
    for conv_p, bn_p, act, inp, res, up, out in steps:
        conv = m.get_submodule(conv_p)
        w = conv.weight.detach().float()
        e = weight_exponent(w)
        w_hi, w_lo = split_planes(w * 2.0 ** e)
        a_hi, a_lo = split_planes(look(inp))
        cv = lambda a, b: F.conv2d(a, b, stride=conv.stride, padding=conv.padding)
        hi_lo = cv(a_hi, w_lo)
        lo_hi = cv(a_lo, w_hi)
        if defect == "remainder_hi_only":
            _, rem = conv_layout(w.shape[1])
            assert rem, f"{conv_p}: Cin {w.shape[1]} has no remainder channels"
            keep = torch.ones(w.shape[1], dtype=torch.float64, device=w.device)
            keep[-rem:] = 0
            hi_lo = cv(a_hi, w_lo * keep.view(1, -1, 1, 1))
            lo_hi = cv(a_lo * keep.view(1, -1, 1, 1), w_hi)
        acc = cv(a_hi, w_hi) + (0 if defect == "hi_lo_dropped" else hi_lo) + (0 if defect == "lo_hi_dropped" else lo_hi)
        acc = acc * 2.0 ** (-e)
        if bn_p is not None:
            scale, shift = _bn(m.get_submodule(bn_p), torch.float64)
            acc = acc * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
        if res is not None:
            acc = acc + look(res)
        if up is not None:
            acc = acc + F.interpolate(look(up), scale_factor=2.0, mode="bilinear", align_corners=True)
        if act == "relu":
            acc = F.relu(acc)
        elif act == "leaky":
            acc = F.leaky_relu(acc, 0.01)
        y = acc
        mid[out] = store_split(y, defect)
    return mid[steps[-1][6]]


# ------------------------------------------------------------------------------------------------ rules
STORE_TERM = 2.0 ** -22   # hi + lo storage of the output: x = hi + lo to 2^-22 of |x|
FP16_STORE_TERM = 2.0 ** -11   # one fp16 plane: half an fp16 ulp at the output's scale
FACTOR = 4                # the kernel's error may be this many times the fp32 oracle's
FP16_DIFF_SHARE = 0.01    # share of stored fp16 values allowed to differ from fp16(ref) at all


def _bias(got, ref):
    """mean(sign(ref) (kernel - ref)) / mean|kernel - ref|: -1 when every error shrinks |ref| (truncation), ~0 when
    errors have no preferred sign"""
    d = got - ref
    return ((torch.sign(ref) * d).mean() / d.abs().mean().clamp_min(1e-300)).item()


def split_rule(got, ref, oracle, factor=FACTOR, store_term=STORE_TERM):
    """max|kernel - ref| <= factor max|oracle - ref| + store_term scale (scale = max|ref|) -> (passed, stats)"""
    ek = (got - ref).abs().max().item()
    eo = (oracle.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    bound = factor * eo + store_term * scale
    ratio = ek / bound if bound > 0 else (0.0 if ek == 0 else float("inf"))
    return ek <= bound, {"err_kernel": ek, "err_oracle": eo, "scale": scale, "bound": bound, "ratio": ratio,
                         "kernel_over_oracle": ek / max(eo, 1e-300), "bias": _bias(got, ref)}


def fp16_ulp(x):
    """Spacing of fp16 at the fp16 values x (2^-24 below the normal range)"""
    _, ex = torch.frexp(x)
    return torch.where(x.abs() < 2.0 ** -14, torch.full_like(x, 2.0 ** -24), torch.ldexp(torch.ones_like(x), ex - 11))


def fp16_rule(got, ref, oracle, factor=FACTOR, share=FP16_DIFF_SHARE):
    """Stored fp16 values: |kernel - fp16(ref)| <= ulp(fp16(ref)) + factor max|oracle - ref| everywhere, and at most
    `share` of them differ from fp16(ref) -> (passed, stats)"""
    r16 = ref.half().double()
    ulp = fp16_ulp(r16)
    d = (got - r16).abs()
    eo = (oracle.double() - ref).abs().max().item()
    ratio = (d / (ulp + factor * eo)).max().item()
    differing = (d > 0).double().mean().item()
    stats = {"err_kernel": (got - ref).abs().max().item(), "err_oracle": eo, "scale": ref.abs().max().item(),
             "ratio": ratio, "max_ulps": (d / ulp).max().item(), "share_differing": differing,
             "share_over_1ulp": (d > ulp).double().mean().item(), "bias": _bias(got, ref)}
    return ratio <= 1 and differing <= share, stats
