"""`LoFTR(config)` / `matcher(batch)` -- the drop-in boundary (reference src/loftr/loftr.py:12-81).

Same constructor argument (the lower-case config dict), same sub-module and parameter names (so
`state_dict`s and released checkpoints round-trip), same `forward(data) -> None` contract that
mutates `data` with the reference's output keys.  Everything runs in the hand-written sm_90a kernels behind the
C ABI of include/loftr_b200.h: the ResNet-FPN backbone as implicit-GEMM convolutions on the tensor cores
(`backbone_impl="b200"`, the default for the shipped ResNetFPN_8_2 shape; `"torch"` keeps the PyTorch/cuDNN fp32
forward, which is closer to fp64 -- DESIGN.md §10; `"b200_fp16"` is the opt-in single-pass fp16 variant, faster and
less accurate -- DESIGN.md §15), then position encoding, coarse transformer, coarse
matching, fine windows, fine transformer and fine matching (`match_precision="fp16"`: the opt-in single-pass fp16
products for the transformers and the coarse score matrix -- DESIGN.md §16).
There is no fallback path: without the built library / an H100 the forward raises.

Packed-weight caches.  The kernels read fp16 hi/lo planes packed lazily from the parameters.  The caches are
rebuilt when a parameter is replaced or modified through autograd-visible in-place ops (`_version` / `data_ptr`
change) and are dropped by `load_state_dict`, `.to()/.cuda()/.float()` (`_apply`) and `invalidate_packed()`.
Writes through `.data` (`p.data.copy_(w)`, EMA swaps, `m.weight.data.normal_()`) change neither `_version` nor
`data_ptr`: call `model.invalidate_packed()` after them.  The caches never enter `copy.deepcopy` / `pickle` /
`torch.save(model)` state.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers

import torch
import torch.nn as nn

from . import _lib, geometry
from .backbone import build_backbone

_KIND = {("self", "linear"): _lib.LAYER_SELF, ("cross", "linear"): _lib.LAYER_CROSS,
         ("self", "full"): _lib.LAYER_SELF_FULL, ("cross", "full"): _lib.LAYER_CROSS_FULL}
ATTENTIONS = ("linear", "full")   # reference config: coarse.attention / fine.attention, options ['linear', 'full']
# operand precision of the transformers' and the coarse score matrix's tensor-core products: "split" (hi/lo planes,
# three MMAs per product: the parity path) or "fp16" (the hi planes only, one MMA per product; DESIGN.md §16)
MATCH_PRECISIONS = ("split", "fp16")


def _check_match_precision(precision, who):
    if isinstance(precision, str) and precision in MATCH_PRECISIONS:
        if precision == "fp16":
            _lib.require(_lib.MATCH_FP16_VERSION, f'{who}="fp16"')
        return precision
    raise ValueError(f"{who} must be one of {MATCH_PRECISIONS} (got {precision!r})")


MAX_PAIRS = 65535   # pairs per call: the coarse transformer's attention kernels put a pass's images in grid.z


def check_pairs(n, who):
    """Refuses more than MAX_PAIRS pairs in one call (`who` names the caller), before anything is launched."""
    if n > MAX_PAIRS:
        raise ValueError(f"{who}: {n} pairs exceed the {MAX_PAIRS} pairs of one call (CUDA's grid.z limit); "
                         "split the pair list into calls of at most that many")


GUIDE_KINDS = {"homography": _lib.GUIDE_HOMOGRAPHY, "fundamental": _lib.GUIDE_FUNDAMENTAL}


def check_guide(guide, n, device, thr, who):
    """Validates a guided-matching guide (DESIGN.md §18) for `n` pairs whose features live on `device`, with the
    coarse threshold `thr`, before any launch and without a host sync; `who` names the caller in the messages.
    guide: {"kind": "fundamental" | "homography", "model": float32 CUDA [n, 3, 3], "radius": finite float > 0}
    -> (LB_GUIDE_* kind code, model, radius)."""
    if not isinstance(guide, dict):
        raise TypeError(f"{who}: guide must be a dict with the keys kind, model and radius (got {type(guide).__name__})")
    if set(guide) != {"kind", "model", "radius"}:
        raise ValueError(f"{who}: guide must have exactly the keys kind, model and radius (got {sorted(map(str, guide))})")
    kind, model, radius = guide["kind"], guide["model"], guide["radius"]
    if not isinstance(kind, str) or kind not in GUIDE_KINDS:
        raise ValueError(f"{who}: guide['kind'] must be one of {tuple(GUIDE_KINDS)} (got {kind!r})")
    if not torch.is_tensor(model) or model.dtype != torch.float32:
        raise TypeError(f"{who}: guide['model'] must be a float32 tensor (got "
                        f"{model.dtype if torch.is_tensor(model) else type(model).__name__})")
    if tuple(model.shape) != (n, 3, 3):
        raise ValueError(f"{who}: guide['model'] must be [N, 3, 3] with N = {n} pairs (got {tuple(model.shape)})")
    if model.device != torch.device(device):
        raise ValueError(f"{who}: guide['model'] is on {model.device}, the features on {device}")
    if isinstance(radius, bool) or not isinstance(radius, numbers.Real):
        raise TypeError(f"{who}: guide['radius'] must be a real number (got {type(radius).__name__})")
    if not (math.isfinite(radius) and radius > 0):
        raise ValueError(f"{who}: guide['radius'] must be finite and positive (got {radius!r})")
    if thr < 0:
        raise ValueError(f"{who}: a guide needs match_coarse.thr >= 0 (got {thr}): with thr < 0 the reference's "
                         "mconf != 0 filter would bring back the entries the guide sets to 0")
    _lib.require_entries(_lib.GUIDE_ENTRIES, f"{who}: guided matching")
    return GUIDE_KINDS[kind], model.contiguous(), float(radius)


def check_rectify(model, n, device, who):
    """Validates a rectifying model (data["rectify1"], DESIGN.md §19) for `n` pairs whose image0 lives on `device`,
    before any launch and without a host sync; `who` names the caller in the messages.
    model: float32 CUDA [n, 3, 3], one homography x1 ~ H x0 per pair -> the model as the kernels read it."""
    if not torch.is_tensor(model) or model.dtype != torch.float32:
        raise TypeError(f"{who}: rectify1 must be a float32 tensor (got "
                        f"{model.dtype if torch.is_tensor(model) else type(model).__name__})")
    if tuple(model.shape) != (n, 3, 3):
        raise ValueError(f"{who}: rectify1 must be [N, 3, 3] with N = {n} pairs (got {tuple(model.shape)})")
    if model.device != torch.device(device):
        raise ValueError(f"{who}: rectify1 is on {model.device}, the images on {device}")
    _lib.require_entries(_lib.RECTIFY_ENTRIES, f"{who}: rectified matching")
    if not model.is_cuda:
        raise ValueError(f"{who}: rectify1 must be a CUDA tensor (the warp and the back-mapping run on the GPU)")
    return model.contiguous()


def check_rectify_candidates(cands, n, device, who):
    """Validates the candidates of a rectification search (data["rectify1_candidates"], DESIGN.md §20) for `n` pairs
    whose image0 lives on `device`, before any launch and without a host sync; `who` names the caller in the messages.
    cands: float32 CUDA [n, K, 3, 3], K >= 1 homographies x1 ~ H x0 per pair (each as data["rectify1"]), n * K at most
    65535 -> the candidates as the kernels read them."""
    if not torch.is_tensor(cands) or cands.dtype != torch.float32:
        raise TypeError(f"{who}: rectify1_candidates must be a float32 tensor (got "
                        f"{cands.dtype if torch.is_tensor(cands) else type(cands).__name__})")
    if cands.dim() != 4 or cands.shape[0] != n or tuple(cands.shape[2:]) != (3, 3):
        raise ValueError(f"{who}: rectify1_candidates must be [N, K, 3, 3] with N = {n} pairs (got "
                         f"{tuple(cands.shape)})")
    k = cands.shape[1]
    if k < 1:
        raise ValueError(f"{who}: rectify1_candidates needs at least one candidate per pair (got K = 0)")
    if n * k > 65535:
        raise ValueError(f"{who}: rectify1_candidates holds N * K = {n * k} candidate pairs, more than the warp's "
                         "65535")
    if cands.device != torch.device(device):
        raise ValueError(f"{who}: rectify1_candidates is on {cands.device}, the images on {device}")
    _lib.require_entries(_lib.SEARCH_ENTRIES + _lib.RECTIFY_ENTRIES, f"{who}: the rectification search")
    if not cands.is_cuda:
        raise ValueError(f"{who}: rectify1_candidates must be a CUDA tensor (the warp and the search run on the GPU)")
    return cands.contiguous()


def _warped_input(data, models, k, who):
    """The substituted input of a rectified call (DESIGN.md §19), or of a rectification search with k candidates per
    pair (§20), without a host sync: image0, and image1 of pair b warped onto image0's canvas through models[b * k + j]
    for j < k ([n * k, 3, 3], `check_rectify`), with pair b's scale1 := scale0 and mask1 := mask0 for each of its k
    candidates.  The scales and masks are checked first."""
    from .preprocess import warp_images   # preprocess imports this module
    if ("scale0" in data) != ("scale1" in data):
        raise ValueError(f"{who}: give scale0 and scale1 together")
    if ("mask0" in data) != ("mask1" in data):
        raise ValueError(f"{who}: give mask0 and mask1 together")
    img0, img1 = data["image0"], data["image1"]
    want = (img1.shape[0], img1.shape[2] // 8, img1.shape[3] // 8)
    if "mask1" in data and tuple(data["mask1"].shape) != want:
        raise ValueError(f"{who}: mask1 must be [N, H1/8, W1/8] = {want} (got {tuple(data['mask1'].shape)})")

    def rep(t):   # t[b] for each of pair b's k candidates (expand + copy: no host sync)
        return t if k == 1 or t is None else t.unsqueeze(1).expand(t.shape[0], k, *t.shape[1:]).flatten(0, 1)

    work = {"image0": img0, "image1": warp_images(rep(img1), models, img0.shape[2:], rep(data.get("scale0")),
                                                  rep(data.get("scale1")))}
    if "scale0" in data:
        work["scale0"] = work["scale1"] = rep(data["scale0"])
    if "mask0" in data:
        work["mask0"] = work["mask1"] = rep(data["mask0"])
    return work


def _map_back(data, model, pts, ids, live=None, inside=True):
    """Points of the rectified frame back into image1 through each pair's model (lb_rectify_points, DESIGN.md §19),
    with the image sizes, scales and mask1 of the caller's `data`.  pts [m, 2] f32 (source pixels of image0's frame),
    ids int64 [m] (the pair of each point), model [n, 3, 3] (`check_rectify`), live: None or the int32 device count
    that bounds the points written.  No host sync.
    -> (mapped [m, 2] f32 in source pixels of image1, inside [m] bool or None when not `inside`)."""
    dev = pts.device
    m = pts.shape[0]
    out = torch.empty(m, 2, dtype=torch.float32, device=dev)
    flag = torch.empty(m, dtype=torch.bool, device=dev) if inside else None
    s0, s1, m1 = (None if data.get(k) is None else data[k].to(dev, t).contiguous()
                  for k, t in (("scale0", torch.float32), ("scale1", torch.float32), ("mask1", torch.uint8)))
    pts, ids = pts.contiguous(), ids.contiguous()
    (h0, w0), (h1, w1) = data["image0"].shape[2:], data["image1"].shape[2:]
    _lib.check(_lib.load().lb_rectify_points(
        pts.data_ptr(), ids.data_ptr(), m, _lib.ptr(live), model.data_ptr(), model.shape[0], _lib.ptr(s0),
        _lib.ptr(s1), h0, w0, h1, w1, _lib.ptr(m1), w1 // 8, out.data_ptr(),
        None if flag is None else flag.view(torch.uint8).data_ptr(), _stream(dev)))
    return out, flag


def _stream(ref=None):
    """cudaStream_t of torch's current stream ON THE DEVICE THAT OWNS `ref` (a tensor or torch.device); the library
    binds itself to the device of the buffers it is given, so the stream handle must belong to that device too."""
    dev = ref.device if torch.is_tensor(ref) else ref
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _weights_key(module):
    """(data_ptr, _version) of every parameter and buffer of `module`: changes when one is replaced, moved or modified
    in place (not through `.data`)."""
    return tuple((t.data_ptr(), t._version) for t in (*module.parameters(), *module.buffers()))


class _PackedCache:
    """A packed copy of the weights of `_packed_source()` (by default the module itself), built by `_build()`.
    `_pack()` rebuilds it when `_weights_key` of that module changes.  It is dropped whenever the parameters are
    re-materialised (`_apply`: .to / .cuda / .float / .half) or re-loaded, and by `invalidate_packed()`, and it never
    enters deepcopy / pickle state: it holds ctypes structures with raw device pointers."""
    _packed = None
    _packed_key = None

    def _packed_source(self):
        return self

    def _pack(self):
        key = _weights_key(self._packed_source())
        if self._packed is None or self._packed_key != key:
            with torch.no_grad():
                self._packed = self._build()
            self._packed_key = key
        return self._packed

    def invalidate_packed(self):
        self._packed = self._packed_key = None

    def __getstate__(self):
        return {**super().__getstate__(), "_packed": None, "_packed_key": None}

    def _apply(self, fn, *args, **kwargs):
        self.invalidate_packed()
        return super()._apply(fn, *args, **kwargs)

    def _load_from_state_dict(self, *args, **kwargs):
        self.invalidate_packed()
        return super()._load_from_state_dict(*args, **kwargs)


def _require_eval(module):
    if module.training:
        raise NotImplementedError("loftr_b200 builds the inference path only: call .eval()")


def _require_cuda(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"loftr_b200: `{name}` must live on a CUDA (H100) device; the matching hot path has "
                           "no CPU implementation")


def weight_exponent(w: torch.Tensor) -> int:
    """The power-of-two exponent e of `split_weight`: max|w| * 2^e ~ 2^12, clamped to [-24, 24]."""
    amax = float(w.abs().max())
    e = 0 if amax == 0.0 else int(math.floor(math.log2(4096.0 / amax)))
    return max(min(e, 24), -24)


def split_weight(w: torch.Tensor):
    """Weight matrix -> (hi, lo, acc_scale): planes of w * 2^e with e chosen so that max|w| * 2^e ~ 2^12, and
    acc_scale = 2^-e for the epilogue.  Power-of-two scaling is exact; it moves the `lo` residuals of typical
    (small) weights out of fp16's subnormal range, where they would only carry ~1e-6 relative accuracy."""
    w = w.detach().float().contiguous()
    e = weight_exponent(w)
    hi, lo = split_planes((w * (2.0 ** e)).contiguous())
    return hi, lo, 2.0 ** (-e)


def split_planes(x: torch.Tensor, hi: torch.Tensor | None = None, lo: torch.Tensor | None = None, col0: int = 0):
    """fp32 [rows, cols] -> fp16 hi/lo planes via the library kernel (x ~= hi + lo)."""
    assert x.dim() == 2 and x.dtype == torch.float32
    _require_cuda(x, "x")
    x = x.contiguous()
    rows, cols = x.shape
    if hi is None:
        hi = torch.empty(rows, cols, dtype=torch.float16, device=x.device)
        lo = torch.empty(rows, cols, dtype=torch.float16, device=x.device)
    lib = _lib.load()
    _lib.check(lib.lb_split_planes(x.data_ptr(), rows, cols, x.stride(0), hi.data_ptr(), lo.data_ptr(), hi.stride(0),
                                   col0, _stream(x)))
    return hi, lo


class TensorCoreBackbone(_PackedCache):
    """ResNetFPN_8_2 forward through `lb_backbone_forward` (implicit-GEMM convolutions on wgmma).  Holds no
    parameters of its own: it packs the weights of the PyTorch `ResNetFPN` module it wraps (BatchNorm folded
    with its running statistics = eval mode), lazily and again whenever a parameter or buffer changes.  It is not a
    submodule, so `LoFTR` drops its cache on `_apply` / `load_state_dict`.

    precision: "split" (hi/lo planes, three MMAs per product: the parity path) or "fp16" (`lb_backbone_forward_fp16`:
    single fp16 activations and one MMA per product after the stem; only the hi weight planes fp16(w * 2^e) are
    packed, DESIGN.md §15)."""

    PRECISIONS = ("split", "fp16")

    def __init__(self, torch_backbone, precision="split"):
        if precision not in self.PRECISIONS:
            raise ValueError(f"TensorCoreBackbone: precision must be one of {self.PRECISIONS} (got {precision!r})")
        if precision == "fp16":
            _lib.require(_lib.BACKBONE_FP16_VERSION, 'the fp16 backbone (backbone_impl="b200_fp16")')
        self.m = torch_backbone
        self.precision = precision

    def _packed_source(self):
        return self.m

    @staticmethod
    def supported(torch_backbone) -> bool:
        # feat_c is stored through an fp32 NHWC tensor map, whose row stride (4 * d3 bytes) must be a multiple of 16
        m = torch_backbone
        d3 = m.layer3[0].conv1.out_channels
        return getattr(m, "depth", 0) == 3 and m.conv1.out_channels == 128 and m.layer1[0].conv1.out_channels == 128 \
            and max(m.layer2[0].conv1.out_channels, d3) <= 256 and d3 % 4 == 0

    @staticmethod
    def _fold(bn, cout, device):
        if bn is None:
            return torch.ones(cout, device=device), torch.zeros(cout, device=device)
        scale = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
        shift = bn.bias.detach().float() - bn.running_mean.detach().float() * scale
        return scale.contiguous(), shift.contiguous()

    def _conv(self, conv, bn, keep):
        w = conv.weight.detach().float()                      # [cout, cin, k, k]
        cout, cin, k, _ = w.shape
        lib = _lib.load()
        bk = lib.lb_block_k()
        cbl, rem = C.c_int(), C.c_int()
        _lib.check(lib.lb_conv_layout(cin, C.byref(cbl), C.byref(rem)))
        cmain = cbl.value * bk                                # channels per tap in the main planes
        wt = w.permute(0, 2, 3, 1).reshape(cout, k * k, cin)  # tap-major
        wp = torch.zeros(cout, k * k, cmain, device=w.device)
        wp[:, :, :min(cin, cmain)] = wt[:, :, :cmain]
        planes = [wp.reshape(cout, k * k * cmain)]
        if rem.value:                                         # channels cmain .. cin-1 of every tap, padded to 16
            wr = torch.zeros(cout, k * k, 16, device=w.device)
            wr[:, :, :rem.value] = wt[:, :, cmain:]
            planes.append(wr.reshape(cout, k * k * 16))
        # one power-of-two scale for both plane sets (they feed the same accumulator)
        wcat = torch.cat(planes, 1)
        if self.precision == "fp16":
            # the hi plane of split_weight, fp16(w * 2^e) rounded to nearest even (the scaling is exact); no lo plane
            e = weight_exponent(wcat)
            hi, lo, acc_scale = (wcat * (2.0 ** e)).half(), None, 2.0 ** (-e)
        else:
            hi, lo, acc_scale = split_weight(wcat)
        nmain = k * k * cmain
        part = lambda t, cols: None if t is None else t[:, cols].contiguous()
        hi_m, lo_m = part(hi, slice(0, nmain)), part(lo, slice(0, nmain))
        hi_r = lo_r = None
        if rem.value:
            hi_r, lo_r = part(hi, slice(nmain, None)), part(lo, slice(nmain, None))
        scale, shift = self._fold(bn, cout, w.device)
        scale = (scale * acc_scale).contiguous()   # y = acc * (2^-e * bn_scale) + bn_shift
        keep += [hi_m, lo_m, hi_r, lo_r, scale, shift]
        return _lib.LbConvWeights(hi_m.data_ptr(), _lib.ptr(lo_m), _lib.ptr(hi_r), _lib.ptr(lo_r), scale.data_ptr(),
                                  shift.data_ptr(), cin, cout, k, conv.stride[0])

    def _build(self):
        m = self.m
        keep = []
        w = _lib.LbBackboneWeights()
        stem = m.conv1.weight.detach().float().reshape(m.conv1.out_channels, 49).t().contiguous()
        sc, sh = self._fold(m.bn1, m.conv1.out_channels, stem.device)
        keep += [stem, sc, sh]
        w.stem_wt, w.stem_scale, w.stem_shift, w.stem_cout = stem.data_ptr(), sc.data_ptr(), sh.data_ptr(), stem.shape[1]
        for name, layer in (("l1", m.layer1), ("l2", m.layer2), ("l3", m.layer3)):
            arr = getattr(w, name)
            for bi, blk in enumerate(layer):
                arr[2 * bi] = self._conv(blk.conv1, blk.bn1, keep)
                arr[2 * bi + 1] = self._conv(blk.conv2, blk.bn2, keep)
            if layer[0].downsample is not None:
                setattr(w, name + "_down", self._conv(layer[0].downsample[0], layer[0].downsample[1], keep))
        w.l3_out = self._conv(m.layer3_outconv, None, keep)
        w.l2_out = self._conv(m.layer2_outconv, None, keep)
        w.l2_out2[0] = self._conv(m.layer2_outconv2[0], m.layer2_outconv2[1], keep)
        w.l2_out2[1] = self._conv(m.layer2_outconv2[3], None, keep)
        w.l1_out = self._conv(m.layer1_outconv, None, keep)
        w.l1_out2[0] = self._conv(m.layer1_outconv2[0], m.layer1_outconv2[1], keep)
        w.l1_out2[1] = self._conv(m.layer1_outconv2[3], None, keep)
        return w, keep

    @torch.no_grad()
    def __call__(self, images):
        """images [N, 1, H, W] fp32 (CUDA) -> (feat_c NHWC [N, H/8, W/8, C3], feat_f NHWC [N, H/2, W/2, C1])."""
        _require_cuda(images, "images")
        lib = _lib.load()
        w, _ = self._pack()
        images = images.float().contiguous()
        n, _, h, wd = images.shape
        c3, c1 = self.m.layer3_outconv.out_channels, self.m.layer1_outconv2[3].out_channels
        feat_c = torch.empty(n, h // 8, wd // 8, c3, dtype=torch.float32, device=images.device)
        feat_f = torch.empty(n, h // 2, wd // 2, c1, dtype=torch.float32, device=images.device)
        fp16 = self.precision == "fp16"
        ws_bytes = lib.lb_backbone_workspace_bytes_fp16 if fp16 else lib.lb_backbone_workspace_bytes
        forward = lib.lb_backbone_forward_fp16 if fp16 else lib.lb_backbone_forward
        nbytes = ws_bytes(C.byref(w), n, h, wd)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=images.device)
        _lib.check(forward(C.byref(w), images.data_ptr(), n, h, wd, feat_c.data_ptr(), feat_f.data_ptr(), ws.data_ptr(),
                           nbytes, _stream(images)))
        return feat_c, feat_f


class PositionEncodingSine(nn.Module):
    """Sinusoidal 2-D position encoding table (reference position_encoding.py:6-42); the add itself is
    fused into the coarse prologue kernel."""

    def __init__(self, d_model, max_shape=(256, 256), temp_bug_fix=True):
        super().__init__()
        pe = torch.zeros((d_model, *max_shape))
        y_position = torch.ones(max_shape).cumsum(0).float().unsqueeze(0)
        x_position = torch.ones(max_shape).cumsum(1).float().unsqueeze(0)
        k = torch.arange(0, d_model // 2, 2).float()
        if temp_bug_fix:
            div_term = torch.exp(k * (-math.log(10000.0) / (d_model // 2)))
        else:  # the historical variant kept for old checkpoints (issue #41 of the reference)
            div_term = torch.exp(k * (-math.log(10000.0) / d_model // 2))
        div_term = div_term[:, None, None]
        pe[0::4] = torch.sin(x_position * div_term)
        pe[1::4] = torch.cos(x_position * div_term)
        pe[2::4] = torch.sin(y_position * div_term)
        pe[3::4] = torch.cos(y_position * div_term)
        self.register_buffer("pe", pe.unsqueeze(0), persistent=False)  # [1, C, H, W]

    def forward(self, x):
        return x + self.pe[:, :, :x.size(2), :x.size(3)]


class LoFTREncoderLayer(nn.Module):
    """Parameter holder with the reference's names/shapes (transformer.py:8-33).  `attention` ('linear' | 'full')
    selects the attention kernels; both kinds have the same parameters."""

    def __init__(self, d_model, nhead, attention="linear"):
        super().__init__()
        if attention not in ATTENTIONS:
            raise ValueError(f"attention must be one of {ATTENTIONS} (got {attention!r})")
        self.attention = attention
        self.dim = d_model // nhead
        self.nhead = nhead
        self.q_proj = nn.Linear(d_model, d_model, bias=False)
        self.k_proj = nn.Linear(d_model, d_model, bias=False)
        self.v_proj = nn.Linear(d_model, d_model, bias=False)
        self.merge = nn.Linear(d_model, d_model, bias=False)
        self.mlp = nn.Sequential(nn.Linear(d_model * 2, d_model * 2, bias=False), nn.ReLU(True),
                                 nn.Linear(d_model * 2, d_model, bias=False))
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)


class _TokenState:
    """Device buffers of one transformer run: fp32 master + fp16 planes ([rows, 2C] cat buffer)."""

    def __init__(self, rows0, rows1, c, device):
        rows = rows0 + rows1
        self.rows0, self.rows1, self.c = rows0, rows1, c
        self.x = torch.empty(rows, c, dtype=torch.float32, device=device)
        self.cat_hi = torch.empty(rows, 2 * c, dtype=torch.float16, device=device)
        self.cat_lo = torch.empty(rows, 2 * c, dtype=torch.float16, device=device)

    def sides(self, n, group_rows0, group_rows1):
        """fp32 master as views of the two sets: [n, group_rows0, C], [n, group_rows1, C]."""
        return self.x[: self.rows0].view(n, group_rows0, self.c), self.x[self.rows0:].view(n, group_rows1, self.c)


class LocalFeatureTransformer(_PackedCache, nn.Module):
    """Interleaved self/cross encoder with linear or full (softmax) attention (reference transformer.py:61-101).

    precision (read-only after construction): "split" or "fp16" (`lb_transformer_forward_fp16`: every tensor-core
    product reads the hi planes only; the same packed weights and token state, DESIGN.md §16)."""

    def __init__(self, config, precision="split"):
        super().__init__()
        self._precision = _check_match_precision(precision, "LocalFeatureTransformer: precision")
        self.config = config
        self.d_model = config["d_model"]
        self.nhead = config["nhead"]
        self.layer_names = list(config["layer_names"])
        self.layers = nn.ModuleList([LoFTREncoderLayer(config["d_model"], config["nhead"], config["attention"])
                                     for _ in self.layer_names])
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)

    @property
    def precision(self):
        return self._precision

    # -- weight packing: fp16 hi/lo planes of the [out, in] matrices
    def _build(self):
        keep = []
        arr = (_lib.LbEncoderLayerWeights * len(self.layers))()
        for i, layer in enumerate(self.layers):
            wqkv = torch.cat([layer.q_proj.weight, layer.k_proj.weight, layer.v_proj.weight], 0).float()
            scaled = [split_weight(wqkv), split_weight(layer.merge.weight), split_weight(layer.mlp[0].weight),
                      split_weight(layer.mlp[2].weight)]
            planes = [(h, l) for h, l, _ in scaled]
            lns = [layer.norm1.weight, layer.norm1.bias, layer.norm2.weight, layer.norm2.bias]
            lns = [t.detach().float().contiguous() for t in lns]
            w = arr[i]
            c, d = self.d_model, self.d_model // self.nhead
            if d == 32 and c == 256 and layer.attention == "linear":
                # fused k|v projection: k and v rows regrouped in blocks of 4 heads (128 rows)
                idx = torch.cat([torch.arange(c + blk * 128, c + blk * 128 + 128).repeat(1) if part == 0 else
                                 torch.arange(2 * c + blk * 128, 2 * c + blk * 128 + 128)
                                 for blk in range(c // 128) for part in (0, 1)]).to(planes[0][0].device)
                wkv = (planes[0][0][idx].contiguous(), planes[0][1][idx].contiguous())
                planes.append(wkv)
                w.wkv_hi, w.wkv_lo = wkv[0].data_ptr(), wkv[1].data_ptr()
            keep.append((planes, lns))
            (w.wqkv_hi, w.wqkv_lo), (w.wm_hi, w.wm_lo), (w.w1_hi, w.w1_lo), (w.w2_hi, w.w2_lo) = [
                (h.data_ptr(), l.data_ptr()) for h, l in planes[:4]]
            w.ln1_g, w.ln1_b, w.ln2_g, w.ln2_b = [t.data_ptr() for t in lns]
            w.s_qkv, w.s_m, w.s_1, w.s_2 = [sc for _, _, sc in scaled]
        kinds = (C.c_int * len(self.layers))(*[_KIND[n, layer.attention] for n, layer in zip(self.layer_names,
                                                                                              self.layers)])
        return arr, kinds, keep

    def run(self, state: _TokenState, n_groups, group_rows0, group_rows1, mask_u8=None, live=None):
        """In-place transformer over a prepared token state (used by LoFTR.forward).  `live` (fine windows only): an
        int32 device count; `n_groups` is then the capacity and only the first min(live, n_groups) windows of each set
        are computed."""
        if any(layer.attention == "full" for layer in self.layers):
            _lib.require(_lib.FULL_ATTENTION_VERSION, "full attention")   # an older library rejects the layer kinds
        lib = _lib.load()
        st = _lib.LbTransformerState(state.x.data_ptr(), state.cat_hi.data_ptr(), state.cat_lo.data_ptr(),
                                     _lib.ptr(mask_u8), n_groups, group_rows0, group_rows1, _lib.ptr(live))
        arr, kinds, _ = self._pack()
        nbytes = lib.lb_transformer_workspace_bytes(self.d_model, self.nhead, n_groups, group_rows0, group_rows1)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=state.x.device)
        fwd = lib.lb_transformer_forward_fp16 if self._precision == "fp16" else lib.lb_transformer_forward
        _lib.check(fwd(arr, kinds, len(self.layers), self.d_model, self.nhead, C.byref(st), ws.data_ptr(), nbytes,
                       _stream(state.x)))

    @torch.no_grad()
    def forward(self, feat0, feat1, mask0=None, mask1=None):
        """feat0 [N, L, C], feat1 [N, S, C] (+ optional bool masks [N, L], [N, S]) -> updated features."""
        assert self.d_model == feat0.size(2), "the feature number of src and transformer must be equal"
        if self.d_model // self.nhead == 32:   # the coarse shape: one group per pair (the fine one has no such limit)
            check_pairs(feat0.shape[0], "LocalFeatureTransformer")
        _require_cuda(feat0, "feat0")
        n, l, c = feat0.shape
        s = feat1.shape[1]
        state = _TokenState(n * l, n * s, c, feat0.device)
        state.x[: n * l] = feat0.reshape(n * l, c)
        state.x[n * l:] = feat1.reshape(n * s, c)
        split_planes(state.x, state.cat_hi, state.cat_lo, 0)
        mask = None
        if mask0 is not None:
            mask = torch.cat([mask0.reshape(-1), mask1.reshape(-1)]).to(torch.uint8).contiguous()
        self.run(state, n, l, s, mask)
        return state.x[: n * l].view(n, l, c).clone(), state.x[n * l:].view(n, s, c).clone()


class CoarseMatching(nn.Module):
    """Dual-softmax / Sinkhorn coarse matching with mutual-nearest selection
    (reference coarse_matching.py:59-261, eval path).

    config["max_matches_per_pair"] (optional, not a reference key): None or absent keeps every match; an int k >= 1
    keeps, within each pair, the k matches with the largest mconf (a tie at the k-th value goes to the smaller row
    index i), selected on the device before the fine stage.  The list stays in ascending (b, i) order.  The attribute
    `max_matches_per_pair` may be changed later; it is validated the same way.

    precision (read-only after construction): "split" or "fp16" (`lb_coarse_match_fp16`: every pass computes the score
    matrix from the hi planes of the features, one MMA per product; DESIGN.md §16)."""

    def __init__(self, config, precision="split"):
        super().__init__()
        self._precision = _check_match_precision(precision, "CoarseMatching: precision")
        self.config = config
        self.max_matches_per_pair = config.get("max_matches_per_pair")
        self.thr = config["thr"]
        self.border_rm = config["border_rm"]
        self.train_coarse_percent = config["train_coarse_percent"]
        self.train_pad_num_gt_min = config["train_pad_num_gt_min"]
        self.match_type = config["match_type"]
        if self.match_type == "dual_softmax":
            self.temperature = config["dsmax_temperature"]
        elif self.match_type == "sinkhorn":
            self.bin_score = nn.Parameter(torch.tensor(config["skh_init_bin_score"], requires_grad=True))
            self.skh_iters = config["skh_iters"]
            self.skh_prefilter = config["skh_prefilter"]
        else:
            raise NotImplementedError()

    @property
    def precision(self):
        return self._precision

    @property
    def max_matches_per_pair(self):
        return self._max_per_pair

    @max_matches_per_pair.setter
    def max_matches_per_pair(self, k):
        if k is not None and (isinstance(k, bool) or not isinstance(k, numbers.Integral) or k < 1):
            raise ValueError(f"match_coarse.max_matches_per_pair must be None or an int >= 1 (got {k!r})")
        self._max_per_pair = None if k is None else int(k)

    @staticmethod
    def default_capacity(n, L, S, masked, max_per_pair=None):
        """Exact bound on the number of coarse matches: mutual nearest neighbours pair each row with at most one
        column, so n*min(L, S) without masks (n*L with masks, as padding may leave columns unmatched); with a per-pair
        cap k, n*min(k, that per-pair bound)."""
        per_pair = min(L, S) if not masked else L
        if max_per_pair is not None:
            per_pair = min(per_pair, max_per_pair)
        return max(n * per_pair, 1)

    def run(self, hi, lo, ld, n, L, S, c, data, mask_u8_0=None, mask_u8_1=None, static=False, capacity=None,
            search=None):
        """Planes of feat_c0 (rows [0, n*L)) / feat_c1 (rows [n*L, ...)) -> coarse match keys in `data`.
        data["guide"] (optional, `check_guide`): guided matching through lb_coarse_match_guided (DESIGN.md §18).
        search: None, or K (the rectification search, DESIGN.md §20): the n "pairs" are n / K pairs of K candidates
        each, and lb_coarse_match_search keeps only each pair's winning candidate's matches.  It writes
        data["rectify1_counts"] [n / K, K] int32 and data["rectify1_choice"] [n / K] int64; b_ids hold candidate ids and
        the default capacity is the bound of n / K pairs.
        Eager (static=False): the lists are trimmed to the match count, read with one host sync.
        Static: no host sync; the match keys are buffers of `capacity` entries (default_capacity when None; entries at
        or past min(count, capacity) unspecified) and data["num_matches"] is the int32 device count [1].  Static needs
        thr >= 0, where the `mconf != 0` filter keeps every row.
        -> the device count when static (the live bound of the fine stage), else None."""
        _require_eval(self)
        k = self.max_matches_per_pair
        if k is not None:
            _lib.require(_lib.MATCH_CAP_VERSION, "match_coarse.max_matches_per_pair")
        lib = _lib.load()
        n_out = n if search is None else n // search   # pairs whose matches the list can hold
        cap = int(capacity) if capacity is not None else self.default_capacity(n_out, L, S, mask_u8_0 is not None, k)
        dev = hi.device
        b_ids = torch.empty(cap, dtype=torch.int64, device=dev)
        i_ids = torch.empty(cap, dtype=torch.int64, device=dev)
        j_ids = torch.empty(cap, dtype=torch.int64, device=dev)
        mconf = torch.empty(cap, dtype=torch.float32, device=dev)
        mk0 = torch.empty(cap, 2, dtype=torch.float32, device=dev)
        mk1 = torch.empty(cap, 2, dtype=torch.float32, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        a, keep, guide = self._args(hi, lo, ld, n, L, S, c, data, mask_u8_0, mask_u8_1)
        a.capacity = cap
        a.b_ids, a.i_ids, a.j_ids = b_ids.data_ptr(), i_ids.data_ptr(), j_ids.data_ptr()
        a.mconf, a.mkpts0_c, a.mkpts1_c, a.count = mconf.data_ptr(), mk0.data_ptr(), mk1.data_ptr(), count.data_ptr()
        conf = None
        if self.config.get("return_conf_matrix", False):   # opt-in: 4*L*S bytes per pair, training-loss input only
            conf = torch.empty(n, L, S, dtype=torch.float32, device=dev)
            a.conf_matrix = conf.data_ptr()
        nbytes = lib.lb_coarse_match_workspace_bytes(n, L, S)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        if search is not None:   # 0: no cap
            _lib.require_entries(_lib.SEARCH_ENTRIES, "the rectification search")
            counts = torch.empty(n_out, search, dtype=torch.int32, device=dev)
            choice = torch.empty(n_out, dtype=torch.int64, device=dev)
            srch = _lib.LbCoarseSearch(search, counts.data_ptr(), choice.data_ptr())
            _lib.check(lib.lb_coarse_match_search(C.byref(a), C.byref(srch), 0 if k is None else min(k, L),
                                                  int(self._precision == "fp16"), ws.data_ptr(), nbytes, _stream(hi)))
            data.update({"rectify1_counts": counts, "rectify1_choice": choice})
        elif guide is not None:   # 0: no cap
            _lib.check(lib.lb_coarse_match_guided(C.byref(a), C.byref(guide), 0 if k is None else min(k, L),
                                                  int(self._precision == "fp16"), ws.data_ptr(), nbytes, _stream(hi)))
        elif self._precision == "fp16":   # 0: no cap
            _lib.check(lib.lb_coarse_match_fp16(C.byref(a), 0 if k is None else min(k, L), ws.data_ptr(), nbytes,
                                                _stream(hi)))
        elif k is None:
            _lib.check(lib.lb_coarse_match(C.byref(a), ws.data_ptr(), nbytes, _stream(hi)))
        else:   # k >= L keeps every match; min() keeps the argument within a C int
            _lib.check(lib.lb_coarse_match_capped(C.byref(a), min(k, L), ws.data_ptr(), nbytes, _stream(hi)))
        m = cap
        if not static:
            m = int(count.item())  # the one host sync of the coarse stage (sizes the match list)
            if m > cap:
                raise RuntimeError(f"loftr_b200: {m} coarse matches exceed the buffer capacity {cap}")
            b_ids, i_ids, j_ids, mconf, mk0, mk1 = b_ids[:m], i_ids[:m], j_ids[:m], mconf[:m], mk0[:m], mk1[:m]
        data.update({"b_ids": b_ids, "i_ids": i_ids, "j_ids": j_ids})
        if conf is not None:
            data["conf_matrix"] = conf
        if self.thr >= 0:  # conf > thr >= 0  =>  the reference's `mconf != 0` filter keeps everything
            data.update({"gt_mask": torch.zeros(m, dtype=torch.bool, device=dev), "m_bids": b_ids,
                         "mkpts0_c": mk0, "mkpts1_c": mk1, "mconf": mconf})
        else:
            nz = mconf != 0
            data.update({"gt_mask": ~nz, "m_bids": b_ids[nz], "mkpts0_c": mk0[nz], "mkpts1_c": mk1[nz],
                         "mconf": mconf[nz]})
        if static:
            data["num_matches"] = count
            return count
        return None

    def _args(self, hi, lo, ld, n, L, S, c, data, mask_u8_0, mask_u8_1):
        """LbCoarseMatchArgs of the coarse stage without its match-list outputs -> (args, tensors it points into,
        LbCoarseGuide of data["guide"] or None; None as well when there is no pair to match)."""
        dev = hi.device
        a = _lib.LbCoarseMatchArgs()
        esz = hi.element_size()
        a.f0_hi, a.f0_lo = hi.data_ptr(), lo.data_ptr()
        a.f1_hi, a.f1_lo = hi.data_ptr() + n * L * ld * esz, lo.data_ptr() + n * L * ld * esz
        a.ld, a.n_pairs, a.L, a.S, a.C = ld, n, L, S, c
        (a.h0c, a.w0c), (a.h1c, a.w1c) = data["hw0_c"], data["hw1_c"]
        a.match_type = _lib.MATCH_DUAL_SOFTMAX if self.match_type == "dual_softmax" else _lib.MATCH_SINKHORN
        a.temperature = float(getattr(self, "temperature", 1.0))
        a.thr, a.border_rm = float(self.thr), int(self.border_rm)
        keep = []
        if self.match_type == "sinkhorn":
            bs = self.bin_score.detach().float().reshape(1).contiguous()
            keep.append(bs)
            a.bin_score, a.skh_iters, a.skh_prefilter = bs.data_ptr(), int(self.skh_iters), int(bool(self.skh_prefilter))
        a.mask0, a.mask1 = _lib.ptr(mask_u8_0), _lib.ptr(mask_u8_1)
        a.img_scale = data["hw0_i"][0] / data["hw0_c"][0]
        if "scale0" in data:
            s0 = data["scale0"].to(dev, torch.float32).contiguous()
            s1 = data["scale1"].to(dev, torch.float32).contiguous()
            keep += [s0, s1]
            a.scale0, a.scale1 = s0.data_ptr(), s1.data_ptr()
        guide = None
        if data.get("guide") is not None and n > 0:
            kind, model, radius = check_guide(data["guide"], n, dev, self.thr, "CoarseMatching")
            keep.append(model)
            guide = _lib.LbCoarseGuide(kind, model.data_ptr(), radius)
        return a, keep, guide

    def query(self, hi, lo, ld, n, L, S, c, data, mask_u8_0, mask_u8_1, points0, valid0=None, side=0, ws=None,
              reuse=False):
        """The coarse stage for caller-given image0 points (LoFTR.match_points, DESIGN.md §17): planes as `run`,
        points0 [n, Q, 2] f32 and valid0 (None or bool [n, Q]) on the device, validated by the caller.  No host sync.
        data["guide"] (optional, `check_guide`): the queries are answered on the guided coarse quantities through
        lb_coarse_query_guided (DESIGN.md §21).
        -> dict of the per-query outputs (q_i_ids, q_j_ids, qconf, qmutual, qvalid, qinside [n, Q]; qpts0_f, qpts1_c
        [n, Q, 2]) and of what the fine stage reads: "centres" int32 [2, n*Q, 2] and "win_ids" int64 [3, n*Q].
        The per-pair cap (max_matches_per_pair) is not applied.
        side: 0, or 1 when points0 / valid0 are image1 points (DESIGN.md §22, lb_coarse_query_side): the outputs are
        then qpts1_f (the snapped query) and qpts0_c (the image0 window centre) in place of qpts0_f / qpts1_c.
        ws: None, or a uint8 device tensor of lb_coarse_match_workspace_bytes(n, L, S) bytes to use as the workspace.
        reuse: ws holds what a preceding query on the same planes and `data` computed, and only the query kernel runs
        (lb_coarse_query_reuse): no score pass."""
        _require_eval(self)
        _lib.require_entries(_lib.POINTS_ENTRIES, "match_points")
        lib = _lib.load()
        dev = hi.device
        q = points0.shape[1]
        nq = n * q
        snap, centre = ("qpts0_f", "qpts1_c") if side == 0 else ("qpts1_f", "qpts0_c")
        out = {"q_i_ids": torch.empty(n, q, dtype=torch.int64, device=dev),
               "q_j_ids": torch.empty(n, q, dtype=torch.int64, device=dev),
               "qconf": torch.empty(n, q, dtype=torch.float32, device=dev),
               "qmutual": torch.empty(n, q, dtype=torch.bool, device=dev),
               "qvalid": torch.empty(n, q, dtype=torch.bool, device=dev),
               "qinside": torch.empty(n, q, dtype=torch.bool, device=dev),
               snap: torch.empty(n, q, 2, dtype=torch.float32, device=dev),
               centre: torch.empty(n, q, 2, dtype=torch.float32, device=dev),
               "centres": torch.empty(2, nq, 2, dtype=torch.int32, device=dev),
               "win_ids": torch.empty(3, nq, dtype=torch.int64, device=dev)}
        a, keep, guide = self._args(hi, lo, ld, n, L, S, c, data, mask_u8_0, mask_u8_1)
        qa = _lib.LbCoarseQueryArgs()
        points0 = points0.contiguous()
        keep.append(points0)
        qa.Q, qa.points0 = q, points0.data_ptr()
        if valid0 is not None:
            valid0 = valid0.contiguous().view(torch.uint8)
            keep.append(valid0)
            qa.valid0 = valid0.data_ptr()
        s = "01"[side]   # the queried image's sizes
        (qa.H0, qa.W0), (qa.Hf0, qa.Wf0) = data[f"hw{s}_i"], data[f"hw{s}_f"]
        qa.stride = data[f"hw{s}_f"][0] // data[f"hw{s}_c"][0]
        qa.fine_scale = data[f"hw{s}_i"][0] / data[f"hw{s}_f"][0]
        qa.i_ids, qa.j_ids, qa.conf = out["q_i_ids"].data_ptr(), out["q_j_ids"].data_ptr(), out["qconf"].data_ptr()
        qa.mutual, qa.valid, qa.inside = (out[k].data_ptr() for k in ("qmutual", "qvalid", "qinside"))
        qa.centres, qa.win_ids = out["centres"].data_ptr(), out["win_ids"].data_ptr()
        qa.pts0_f, qa.pts1_c = out[snap].data_ptr(), out[centre].data_ptr()
        nbytes = lib.lb_coarse_match_workspace_bytes(n, L, S)
        if ws is None:
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        planes = 1 if self._precision == "fp16" else 2
        if reuse:
            _lib.check(lib.lb_coarse_query_reuse(C.byref(a), C.byref(qa), side, ws.data_ptr(), ws.numel(), _stream(hi)))
        elif side:
            _lib.check(lib.lb_coarse_query_side(C.byref(a), C.byref(qa), None if guide is None else C.byref(guide),
                                                side, planes, ws.data_ptr(), ws.numel(), _stream(hi)))
        elif guide is not None:
            _lib.require_entries(_lib.BANK_POINTS_ENTRIES, "guided point queries")
            _lib.check(lib.lb_coarse_query_guided(C.byref(a), C.byref(qa), C.byref(guide), planes, ws.data_ptr(),
                                                  nbytes, _stream(hi)))
        else:
            _lib.check(lib.lb_coarse_query(C.byref(a), C.byref(qa), planes, ws.data_ptr(), nbytes, _stream(hi)))
        return out

    @torch.no_grad()
    def forward(self, feat_c0, feat_c1, data, mask_c0=None, mask_c1=None):
        """Reference signature (coarse_matching.py:87): feat_c0 [N, L, C], feat_c1 [N, S, C], masks [N, L]/[N, S]."""
        _require_cuda(feat_c0, "feat_c0")
        n, L, c = feat_c0.shape
        S = feat_c1.shape[1]
        x = torch.cat([feat_c0.reshape(n * L, c), feat_c1.reshape(n * S, c)], 0).float().contiguous()
        hi, lo = split_planes(x)
        m0 = mask_c0.reshape(-1).to(torch.uint8).contiguous() if mask_c0 is not None else None
        m1 = mask_c1.reshape(-1).to(torch.uint8).contiguous() if mask_c1 is not None else None
        self.run(hi, lo, c, n, L, S, c, data, m0, m1)


class FinePreprocess(_PackedCache, nn.Module):
    """Window gather + coarse-feature merge (reference fine_preprocess.py:7-59)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.cat_c_feat = config["fine_concat_coarse_feat"]
        self.W = config["fine_window_size"]
        d_model_c = config["coarse"]["d_model"]
        d_model_f = config["fine"]["d_model"]
        self.d_model_f = d_model_f
        if not self.cat_c_feat:
            raise NotImplementedError("fine_concat_coarse_feat=False is not built (every shipped config sets True)")
        self.down_proj = nn.Linear(d_model_c, d_model_f, bias=True)
        self.merge_feat = nn.Linear(2 * d_model_f, d_model_f, bias=True)
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.kaiming_normal_(p, mode="fan_out", nonlinearity="relu")

    def _build(self):
        wm = self.merge_feat.weight.detach().float().contiguous()
        hi, lo, msc = split_weight(wm[:, : self.d_model_f])
        return {"wdt": self.down_proj.weight.detach().float().t().contiguous(),
                "bd": self.down_proj.bias.detach().float().contiguous(),
                "wm2t": wm[:, self.d_model_f:].t().contiguous(),
                "bm": self.merge_feat.bias.detach().float().contiguous(),
                "wm_hi": hi, "wm_lo": lo, "wm_scale": msc}

    def run(self, feat_f0, feat_f1, feat_c_all, n, L, S, data, live=None, img_idx=None, centres=None):
        """-> _TokenState of the fine transformer (rows: side, match, window position); with M == 0 it has no rows
        and nothing is launched.  M is the length of data["b_ids"].
        `live`: int32 device count; the match keys of `data` are then capacity buffers and only windows below the
        count are gathered (rows keep the capacity layout side*cap*WW + m*WW + k).
        `img_idx`: (idx0, idx1) int32 device tensors [n]: feat_f0 / feat_f1 are then feature banks and pair b's
        windows are read from their images idx0[b] / idx1[b].
        `centres`: (centres, inside) of CoarseMatching.query: the windows are centred on the fine pixels of the int32
        table [2, M, 2] rather than on the cells of i_ids / j_ids, and windows m with inside[m] false are zeros.  With
        `img_idx` as well, they are read from the banks' images (lb_fine_preprocess_centres_indexed)."""
        lib = _lib.load()
        W = self.W
        stride = data["hw0_f"][0] // data["hw0_c"][0]
        data.update({"W": W})
        m = int(data["b_ids"].shape[0])
        cf = self.d_model_f
        dev = feat_f0.device
        state = _TokenState(m * W * W, m * W * W, cf, dev)
        if m == 0:
            return state
        p = self._pack()
        a = _lib.LbFinePreprocessArgs()
        a.feat_f0, a.feat_f1 = feat_f0.data_ptr(), feat_f1.data_ptr()
        a.sn0, a.sc0, a.sh0, a.sw0 = feat_f0.stride()
        a.sn1, a.sc1, a.sh1, a.sw1 = feat_f1.stride()
        a.Hf0, a.Wf0 = feat_f0.shape[2:]
        a.Hf1, a.Wf1 = feat_f1.shape[2:]
        a.w0c, a.w1c = data["hw0_c"][1], data["hw1_c"][1]
        a.stride, a.W, a.Cf, a.Cc = stride, W, cf, feat_c_all.shape[1]
        a.feat_c, a.n_pairs, a.L, a.S, a.M = feat_c_all.data_ptr(), n, L, S, m
        a.b_ids, a.i_ids, a.j_ids = data["b_ids"].data_ptr(), data["i_ids"].data_ptr(), data["j_ids"].data_ptr()
        a.down_wt, a.down_b, a.merge_w2t, a.merge_b = (p["wdt"].data_ptr(), p["bd"].data_ptr(), p["wm2t"].data_ptr(),
                                                       p["bm"].data_ptr())
        a.merge_w_hi, a.merge_w_lo, a.merge_acc_scale = p["wm_hi"].data_ptr(), p["wm_lo"].data_ptr(), p["wm_scale"]
        a.x_f32, a.cat_hi, a.cat_lo = state.x.data_ptr(), state.cat_hi.data_ptr(), state.cat_lo.data_ptr()
        a.M_live = _lib.ptr(live)
        nbytes = lib.lb_fine_preprocess_workspace_bytes(m, W, cf)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        if centres is not None and img_idx is not None:
            _lib.check(lib.lb_fine_preprocess_centres_indexed(
                C.byref(a), centres[0].data_ptr(), centres[1].data_ptr(), img_idx[0].data_ptr(), img_idx[1].data_ptr(),
                ws.data_ptr(), nbytes, _stream(feat_f0)))
        elif centres is not None:
            _lib.check(lib.lb_fine_preprocess_centres(C.byref(a), centres[0].data_ptr(), centres[1].data_ptr(),
                                                      ws.data_ptr(), nbytes, _stream(feat_f0)))
        elif img_idx is None:
            _lib.check(lib.lb_fine_preprocess(C.byref(a), ws.data_ptr(), nbytes, _stream(feat_f0)))
        else:
            _lib.check(lib.lb_fine_preprocess_indexed(C.byref(a), img_idx[0].data_ptr(), img_idx[1].data_ptr(),
                                                      ws.data_ptr(), nbytes, _stream(feat_f0)))
        return state

    @torch.no_grad()
    def forward(self, feat_f0, feat_f1, feat_c0, feat_c1, data):
        """Reference signature (fine_preprocess.py:29) -> (feat_f0_unfold, feat_f1_unfold) [M, WW, C_f]."""
        _require_cuda(feat_f0, "feat_f0")
        n, L, cc = feat_c0.shape
        S = feat_c1.shape[1]
        feat_c_all = torch.cat([feat_c0.reshape(n * L, cc), feat_c1.reshape(n * S, cc)], 0).float().contiguous()
        state = self.run(feat_f0.float(), feat_f1.float(), feat_c_all, n, L, S, data)
        ww = self.W ** 2
        return state.sides(state.rows0 // ww, ww, ww)


class FineMatching(nn.Module):
    """Correlation + soft-argmax refinement (reference fine_matching.py:9-74)."""

    @torch.no_grad()
    def forward(self, feat_f0, feat_f1, data, live=None):
        """`live`: int32 device count; M is then the capacity and only matches below the count are refined."""
        M, WW, Cf = feat_f0.shape
        W = int(math.sqrt(WW))
        scale = data["hw0_i"][0] / data["hw0_f"][0]
        if M == 0:
            assert self.training is False, "M is always >0, when training, see coarse_matching.py"
            data.update({"expec_f": torch.empty(0, 3, device=feat_f0.device),
                         "mkpts0_f": data["mkpts0_c"], "mkpts1_f": data["mkpts1_c"]})
            return
        _require_cuda(feat_f0, "feat_f0")
        lib = _lib.load()
        dev = feat_f0.device
        f0 = feat_f0.float().contiguous()
        f1 = feat_f1.float().contiguous()
        expec = torch.empty(M, 3, dtype=torch.float32, device=dev)
        mk1f = torch.empty(M, 2, dtype=torch.float32, device=dev)
        mk1c = data["mkpts1_c"].float().contiguous()
        if mk1c.shape[0] != M:
            raise RuntimeError("fine matching expects one coarse keypoint per window")
        a = _lib.LbFineMatchArgs()
        a.f0, a.f1, a.W, a.C, a.M = f0.data_ptr(), f1.data_ptr(), W, Cf, M
        a.img_scale = scale
        keep = None
        if "scale0" in data:  # the reference tests 'scale0' but applies scale1 (fine_matching.py:68)
            keep = data["scale1"].to(dev, torch.float32).contiguous()
            a.scale1 = keep.data_ptr()
        a.b_ids, a.mkpts1_c = data["b_ids"].data_ptr(), mk1c.data_ptr()
        a.expec_f, a.mkpts1_f = expec.data_ptr(), mk1f.data_ptr()
        a.M_live = _lib.ptr(live)
        _lib.check(lib.lb_fine_match(C.byref(a), _stream(f0)))
        data.update({"expec_f": expec, "mkpts0_f": data["mkpts0_c"], "mkpts1_f": mk1f})


class LoFTR(nn.Module):
    """Top-level matcher (reference loftr.py:12-81)."""

    def __init__(self, config, backbone_impl="auto", match_precision="split"):
        """backbone_impl: "torch" keeps the PyTorch/cuDNN ResNet-FPN forward (the north_star default scope);
        "b200" runs it as implicit-GEMM convolutions on the tensor cores (SURVEY.md §8(f) rank 1); "auto" picks
        "b200" whenever the configured backbone is the supported ResNetFPN_8_2 shape.  "b200_fp16" (opt-in, never
        picked by "auto") runs the same convolutions with single fp16 activations and one fp16 MMA per product: faster,
        but it does not meet the reference-parity target (DESIGN.md §10, §15).  All are GPU paths.

        match_precision: "split" (the default) computes every tensor-core product of the coarse and fine transformers
        and of the coarse score matrix from hi/lo planes; "fp16" (opt-in) from the hi planes only, one fp16 MMA per
        product: faster, but it does not meet the reference-parity target either (DESIGN.md §16).  Independent of
        backbone_impl, and fixed at construction (read-only attribute `match_precision`)."""
        super().__init__()
        self._match_precision = _check_match_precision(match_precision, "LoFTR: match_precision")
        self.config = config
        # the kernels are built for the shipped shapes; anything else must fail here, not at the first forward
        cc, fc = config["coarse"], config["fine"]
        if (cc["d_model"], cc["nhead"]) != (256, 8):
            raise ValueError(f"loftr_b200 builds the coarse transformer for d_model=256, nhead=8 (got {cc['d_model']}, "
                             f"{cc['nhead']})")
        if (fc["d_model"], fc["nhead"]) != (128, 8):
            raise ValueError(f"loftr_b200 builds the fine transformer for d_model=128, nhead=8 (got {fc['d_model']}, "
                             f"{fc['nhead']})")
        if config["fine_window_size"] ** 2 > 32 or config["fine_window_size"] % 2 == 0:
            raise ValueError("loftr_b200 builds fine windows of odd size with at most 32 cells (fine_window_size <= 5)")
        if config["fine_window_size"] < 3:   # the refinement grid steps by 2 / (W - 1)  [fine_matching.py:50]
            raise ValueError(f"fine_window_size must be 3 or 5 (got {config['fine_window_size']}): a 1-cell window has no "
                             "sub-pixel grid to refine on")
        self.expose_coarse_features = False   # True: forward also writes data['_feat_c0'/'_feat_c1'] (not reference keys)
        self.backbone = build_backbone(config)
        if backbone_impl == "auto":
            backbone_impl = "b200" if TensorCoreBackbone.supported(self.backbone) else "torch"
        if backbone_impl not in ("torch", "b200", "b200_fp16"):
            raise ValueError(backbone_impl)
        if backbone_impl != "torch" and not TensorCoreBackbone.supported(self.backbone):
            raise ValueError("the tensor-core backbone is built for ResNetFPN_8_2 with initial_dim 128, dims <= 256 and "
                             "a layer3 width divisible by 4")
        self.backbone_impl = backbone_impl
        self._tc_backbone = None
        if backbone_impl != "torch":
            precision = "fp16" if backbone_impl == "b200_fp16" else "split"
            self._tc_backbone = TensorCoreBackbone(self.backbone, precision=precision)
        self.pos_encoding = PositionEncodingSine(config["coarse"]["d_model"],
                                                 temp_bug_fix=config["coarse"]["temp_bug_fix"])
        self.loftr_coarse = LocalFeatureTransformer(config["coarse"], precision=match_precision)
        self.coarse_matching = CoarseMatching(config["match_coarse"], precision=match_precision)
        self.fine_preprocess = FinePreprocess(config)
        self.loftr_fine = LocalFeatureTransformer(config["fine"], precision=match_precision)
        self.fine_matching = FineMatching()

    @property
    def match_precision(self):
        return self._match_precision

    @torch.no_grad()
    def forward(self, data):
        """Updates `data` in place with the reference's keys; returns None.
        Inputs: image0/image1 [N, 1, H, W] float32 (H, W divisible by 8), optional mask0/mask1 [N, H/8, W/8],
        optional scale0/scale1 [N, 2], optional guide (guided coarse matching, DESIGN.md §18): {"kind":
        "fundamental" | "homography", "model": float32 [N, 3, 3] on image0's device, one matrix per pair in the
        coordinates of mkpts0_f / mkpts1_f, "radius": pixels of image1, finite and > 0}.  Only cell pairs whose coarse
        keypoints agree with the pair's model within the radius can match, and only they enter the softmax (Sinkhorn)
        normalisers; a pair whose model has a non-finite entry is matched unguided.  Needs match_coarse.thr >= 0.

        Optional rectify1 (rectified matching, DESIGN.md §19): float32 [N, 3, 3] on image0's device, one homography
        x1 ~ H x0 per pair in the coordinates of mkpts0_f / mkpts1_f.  The call then matches image0 against image1
        warped onto image0's canvas through H (`warp_images`; scale1 := scale0, mask1 := mask0) and maps mkpts1_c /
        mkpts1_f back through H into image1; the new key minside1 [M] bool says whether mkpts1_f lies in image1's valid
        area.  expec_f, j_ids and hw1_* describe the rectified frame (image0's grid).  The caller's image1, scale1 and
        mask1 are not replaced.  Not combinable with a guide.

        Optional rectify1_candidates (rectification search, DESIGN.md §20): float32 [N, K, 3, 3] on image0's device,
        K >= 1 homographies per pair as rectify1, N * K <= 65535; `rotation_candidates` gives the four quarter turns.
        Each pair is matched under every candidate (image0's backbone runs once), and only the candidate with the most
        coarse matches (before max_matches_per_pair; ties to the smaller k) is kept, capped and refined.  New keys:
        rectify1_choice [N] int64 (that k), rectify1_counts [N, K] int32 (the coarse match count of every candidate)
        and minside1; every other key is that of a rectify1 call with the chosen candidate, b_ids / m_bids holding pair
        ids (bs is N).  The outputs equal those of the rectified call on the N * K candidate pairs restricted to the
        chosen ones, bit for bit with the tensor-core backbones; with K = 1 they are the rectify1 call's.  Not
        combinable with rectify1 or a guide.

        At most MAX_PAIRS (65535) pairs per call."""
        _require_eval(self)
        check_pairs(data["image0"].shape[0], "forward")
        _require_cuda(data["image0"], "image0")
        if data.get("rectify1_candidates") is not None:
            self._match_searched(data, "forward")
            return
        if data.get("rectify1") is not None:
            self._match_rectified(data, "forward")
            return
        if data.get("guide") is not None:
            check_guide(data["guide"], data["image0"].shape[0], data["image0"].device, self.coarse_matching.thr,
                        "forward")
        self._match_pairs(data, *self._backbone_pairs(data))

    @torch.no_grad()
    def extract_features(self, images, masks=None) -> "ImageFeatures":
        """Runs the configured backbone once on images [K, 1, H, W] (CUDA) -> ImageFeatures, a per-image feature bank
        for `match_features`.  masks: optional [K, H/8, W/8] padding masks (as forward's mask0 / mask1), stored with
        the bank.  Position encoding and the transformers are not applied: they depend on the pair."""
        _require_eval(self)
        _require_cuda(images, "images")
        if images.dim() != 4 or images.shape[1] != 1:
            raise ValueError(f"extract_features: images must be [K, 1, H, W] (got {tuple(images.shape)})")
        if images.shape[0] == 0:
            raise ValueError("extract_features: no images (a feature bank holds at least one)")
        key = self._bank_key()
        feat_c, feat_f = self._backbone(images)
        if masks is not None:
            if tuple(masks.shape) != (images.shape[0], *feat_c.shape[2:]):
                raise ValueError(f"extract_features: masks must be [K, H/8, W/8] = {(images.shape[0], *feat_c.shape[2:])} "
                                 f"(got {tuple(masks.shape)})")
            masks = masks.to(images.device)
        return ImageFeatures(feat_c, feat_f, masks, images.shape[2:], feat_c.shape[2:], feat_f.shape[2:], key)

    @torch.no_grad()
    def match_features(self, feats0, idx0, feats1, idx1, scale0=None, scale1=None, data=None, estimate=None,
                       guide=None):
        """Matches pair b = (image idx0[b] of feats0, image idx1[b] of feats1) for every b of the pair list, from banks
        made by `extract_features` (feats1 may be feats0).  Writes into `data` (a new dict when None) and returns it:
        the keys, dtypes and values `forward` writes for the batch image0 = images idx0 of feats0, image1 = images
        idx1 of feats1, with the banks' masks and the scales gathered the same way.  `m_bids` indexes the pair list.

        idx0, idx1: int32 / int64 tensors [B] on the model's device, each index within its bank.  An empty list gives
        the outputs of a forward with no matches.  scale0 / scale1: optional [K0, 2] / [K1, 2] per-image scales of
        feats0 / feats1 (both or neither).  A bank is tied to the backbone weights it was extracted with: after
        load_state_dict, .to() or a parameter update it raises; extract again.

        estimate: None (the default: nothing else runs and no other key is written), "homography", "fundamental", or
        a dict of `loftr_b200.estimate_geometry` options ("model", "threshold", "iterations", "seed").  The estimator
        then fits that model to each pair's fine matches (mkpts0_f / mkpts1_f) on the GPU and adds
        data["geom_model"] [B, 3, 3], data["geom_inliers"] [M] bool (one flag per match of the list) and
        data["geom_num_inliers"] [B] int32; pair b's RNG key is b.

        guide: None, or forward's data["guide"] with "model" [B, 3, 3] in pair-list order: guided coarse matching
        (DESIGN.md §18).  It combines with `estimate`, which then fits the guided matches; a geom_model of an earlier
        call guides the next one directly (a failed pair's NaN model leaves that pair unguided)."""
        _require_eval(self)
        _lib.require(_lib.FEATURE_BANK_VERSION, "match_features")
        geom = None
        if estimate is not None:
            opts = {"model": estimate} if isinstance(estimate, str) else estimate
            if not isinstance(opts, dict) or not set(opts) <= {"model", "threshold", "iterations", "seed"}:
                raise ValueError("match_features: estimate must be None, 'homography', 'fundamental' or a dict of "
                                 "estimate_geometry options (model, threshold, iterations, seed)")
            geom = dict(zip(("model", "threshold", "iterations", "seed"), geometry.check_options(**opts)))
            _lib.require(_lib.GEOMETRY_VERSION, "match_features(estimate=...)")
        idx0, idx1, dev = self._check_banks(feats0, idx0, feats1, idx1, scale0, scale1, "match_features")
        bs = idx0.numel()
        work = {}   # forward's inputs for this pair list (masks, scales, guide), then every key forward writes
        if guide is not None:
            check_guide(guide, bs, dev, self.coarse_matching.thr, "match_features")
            work["guide"] = guide
        work.update(_bank_inputs(feats0, idx0, feats1, idx1, scale0, scale1, dev, "match_features"))
        work.update(_bank_sizes(bs, feats0, feats1))
        self._match_pairs(work, feats0.feat_c, feats1.feat_c, feats0.feat_f, feats1.feat_f, img_idx=(idx0, idx1))
        if geom is not None:
            (h0, w0), (h1, w1) = feats0.hw_c, feats1.hw_c
            bound = CoarseMatching.default_capacity(1, h0 * w0, h1 * w1, feats0.mask is not None,
                                                    self.coarse_matching.max_matches_per_pair)
            geometry.estimate_on_matches(work, bs, bound, geom)
        out = {} if data is None else data
        out.update({k: v for k, v in work.items() if k not in ("mask0", "mask1", "scale0", "scale1", "guide")})
        return out

    @torch.no_grad()
    def match_points_features(self, feats0, idx0, feats1, idx1, points0=None, valid0=None, scale0=None, scale1=None,
                              data=None, guide=None, *, points1=None, valid1=None, round_trip=False):
        """`match_points` on pairs drawn from feature banks (DESIGN.md §21): pair b is image idx0[b] of feats0 against
        image idx1[b] of feats1, as in `match_features` (feats1 may be feats0; the banks' masks and the per-image
        scales scale0 [K0, 2] / scale1 [K1, 2] are gathered through the indices).  The backbone does not run again, so
        a sequence of frames, or one reference image tracked into many, pays for each image once.

        points0: float32 [B, Q, 2] and valid0: optional bool [B, Q], one row per entry of the pair list, as in
        `match_points` (source pixels when scales are given).  Writes into `data` (a new dict when None) and returns it:
        the keys, dtypes and values `match_points` writes for the stacked batch image0 = images idx0 of feats0, image1 =
        images idx1 of feats1, bit for bit with the tensor-core backbones.

        guide: None, or `match_features`' guide ("model" [B, 3, 3] in pair-list order; a NaN model leaves its pair
        unguided).  The queries are then answered on the guided coarse quantities of DESIGN.md §18: j is the row
        arg-max over the admissible cells, qvalid is the guided flag test, and a row without an admissible, unmasked
        column is not inside.  A query at a guided `match_features` match's mkpts0_c returns that match bit for bit.

        points1 / valid1 (keyword-only, instead of points0 / valid0) and round_trip: as in `match_points` (DESIGN.md
        §22), with the scales of the pair list and under the guide when one is given.

        An empty pair list or Q = 0 gives empty outputs and launches nothing.  The one host sync is the index range
        check of `match_features`."""
        who = "match_points_features"
        _require_eval(self)
        side, points, valid = _query_side(points0, valid0, points1, valid1, round_trip, who)
        _lib.require(_lib.FEATURE_BANK_VERSION, who)
        _lib.require_entries(_lib.POINTS_ENTRIES + _lib.BANK_POINTS_ENTRIES, who)
        if side or round_trip:
            _lib.require_entries(_lib.SIDE_POINTS_ENTRIES, who)
        idx0, idx1, dev = self._check_banks(feats0, idx0, feats1, idx1, scale0, scale1, who)
        bs = idx0.numel()
        _check_query_args(points, valid, bs, who, side)
        _check_devices([(f"points{side}", points)] + ([(f"valid{side}", valid)] if valid is not None else []), dev,
                       "the model", who)
        work = {}   # match_points' inputs for this pair list (masks, scales, guide), then every key it writes
        if guide is not None:
            check_guide(guide, bs, dev, self.coarse_matching.thr, who)
            work["guide"] = guide
        q = points.shape[1]
        work.update(_bank_inputs(feats0, idx0, feats1, idx1, scale0, scale1, dev, who, gather=bool(bs and q)))
        work.update(_bank_sizes(bs, feats0, feats1))
        if bs and q:
            self._match_points(work, points, valid, (feats0.feat_c, feats1.feat_c, feats0.feat_f, feats1.feat_f),
                               (idx0, idx1), side, round_trip)
        else:
            work.update(_query_outputs(bs, q, dev, side, round_trip))
        out = {} if data is None else data
        out.update({k: v for k, v in work.items() if k not in ("mask0", "mask1", "scale0", "scale1", "guide")})
        return out

    def _check_banks(self, feats0, idx0, feats1, idx1, scale0, scale1, who):
        """The bank arguments of match_features / match_points_features (`who`), checked before any launch ->
        (idx0, idx1 as contiguous int32 tensors on the model's device, that device)."""
        key = self._bank_key()
        dev = next(self.parameters()).device
        for name, f in (("feats0", feats0), ("feats1", feats1)):
            if not isinstance(f, ImageFeatures):
                raise TypeError(f"{who}: `{name}` must be the ImageFeatures of extract_features")
            if f.weights_key != key:
                raise RuntimeError(f"{who}: `{name}` was extracted with other backbone weights (load_state_dict, "
                                   ".to() or a parameter update since); extract the features again")
        idx0 = self._pair_index(idx0, "idx0", len(feats0), dev, who)
        idx1 = self._pair_index(idx1, "idx1", len(feats1), dev, who)
        if idx0.shape != idx1.shape:
            raise ValueError(f"{who}: idx0 and idx1 must have the same length ({idx0.numel()} vs {idx1.numel()})")
        check_pairs(idx0.numel(), who)
        if (feats0.mask is None) != (feats1.mask is None):
            raise ValueError(f"{who}: either both banks carry masks or neither (as mask0 / mask1 of forward)")
        if (scale0 is None) != (scale1 is None):
            raise ValueError(f"{who}: give scale0 and scale1 together")
        return idx0, idx1, dev

    @staticmethod
    def _pair_index(idx, name, n_images, dev, who="match_features"):
        """Validated pair -> bank image index as a contiguous int32 tensor on `dev` (one host sync for the range)."""
        if not torch.is_tensor(idx) or idx.dtype not in (torch.int32, torch.int64):
            raise TypeError(f"{who}: `{name}` must be an int32 or int64 tensor (got "
                            f"{idx.dtype if torch.is_tensor(idx) else type(idx).__name__})")
        if idx.device != dev:
            raise ValueError(f"{who}: `{name}` is on {idx.device}, the model on {dev}")
        if idx.dim() != 1:
            raise ValueError(f"{who}: `{name}` must be one-dimensional (got shape {tuple(idx.shape)})")
        if idx.numel():
            lo, hi = torch.stack([idx.min(), idx.max()]).tolist()
            if lo < 0 or hi >= n_images:
                raise IndexError(f"{who}: `{name}` holds indices in [{lo}, {hi}], outside the bank's "
                                 f"[0, {n_images})")
        return idx.to(torch.int32).contiguous()

    def _bank_key(self):
        """What a feature bank depends on: the backbone implementation and its tensors' (data_ptr, _version)."""
        return (self.backbone_impl,) + _weights_key(self.backbone)

    def _backbone(self, images):
        """The configured backbone on [N, 1, H, W] -> (feat_c, feat_f) as [N, C, h, w]; NHWC storage (channels-last
        strides) from the tensor-core backbone, NCHW from the PyTorch one."""
        if self._tc_backbone is not None:
            fc, ff = self._tc_backbone(images)
            return fc.permute(0, 3, 1, 2), ff.permute(0, 3, 1, 2)
        return self.backbone(images)

    @torch.no_grad()
    def forward_static(self, data, capacity=None):
        """Sync-free, static-shape forward: the same inputs and keys as `forward`, without any host synchronisation,
        so that it can be captured by `torch.cuda.graph` (after one eager call, which packs the weights).

        Every input, masks and scales included, must already be on the device.  The match keys (b_ids, i_ids, j_ids,
        m_bids, gt_mask, mconf, mkpts0_c/1_c, mkpts0_f/1_f, expec_f) are fixed-capacity tensors with first dimension
        `capacity`, and data["num_matches"] is an int32 device tensor [1] with the true match count.  The count may
        exceed `capacity`; entries at or past min(count, capacity) are unspecified.  Only windows below the count are
        refined: the fine stage reads the count on the device.

        capacity: defaults to the exact bound of the coarse stage, n*min(L, S) (n*L with masks), or n*min(k, that
        per-pair bound) with match_coarse.max_matches_per_pair = k.  The fine stage keeps about 4.8 KB of state per
        window row, i.e. about 240 KB per match of capacity (about 9.4 GB at batch 8 640x480 without k): a smaller
        capacity trades that memory for the risk of overflow, which stays visible in num_matches.  A capacity of n*k
        never overflows.

        Configurations whose output list depends on the data (match_coarse.thr < 0) raise ValueError.

        data["guide"] (as in `forward`): its model must be on the device as well.  A captured graph bakes in the kind
        and the radius and reads the model from the same tensor at every replay.  data["rectify1"] (as in `forward`):
        a captured graph reads it from the same tensor at every replay as well; minside1 is a capacity buffer too.
        data["rectify1_candidates"] (as in `forward`): read from the same tensor at every replay too; the default
        capacity is the bound of the N pairs, since only the winning candidates' matches are listed."""
        _require_static(self, capacity, "forward_static")
        check_pairs(data["image0"].shape[0], "forward_static")
        dev = None
        for k in ("image0", "image1", "mask0", "mask1", "scale0", "scale1"):
            if k not in data:
                continue
            t = data[k]
            if not torch.is_tensor(t) or not t.is_cuda:
                raise ValueError(f"forward_static: `{k}` must already be a CUDA tensor (copying a host tensor to the "
                                 "device would synchronise)")
            if dev is None:
                dev = t.device
            elif t.device != dev:
                raise ValueError(f"forward_static: `{k}` is on {t.device}, image0 on {dev}")
        if data.get("rectify1_candidates") is not None:
            self._match_searched(data, "forward_static", static=True, capacity=capacity)
            return
        if data.get("rectify1") is not None:
            self._match_rectified(data, "forward_static", static=True, capacity=capacity)
            return
        if data.get("guide") is not None:
            check_guide(data["guide"], data["image0"].shape[0], data["image0"].device, self.coarse_matching.thr,
                        "forward_static")
        self._match_pairs(data, *self._backbone_pairs(data), static=True, capacity=capacity)

    def _rectified(self, data, who):
        """The substituted input of a call with data["rectify1"] (DESIGN.md §19), validated before any launch and
        without a host sync -> (work dict: image0, image1 warped onto image0's canvas, scale1 := scale0 and mask1 :=
        mask0 when given; the model as `check_rectify` returns it)."""
        if data.get("guide") is not None:
            raise ValueError(f"{who}: data['rectify1'] cannot be combined with data['guide']")
        img0 = data["image0"]
        model = check_rectify(data["rectify1"], img0.shape[0], img0.device, who)
        return _warped_input(data, model, 1, who), model

    def _match_rectified(self, data, who, static=False, capacity=None):
        """forward / forward_static with data["rectify1"]: the call on the substituted input, then mkpts1_c / mkpts1_f
        mapped back and minside1; every key the call writes goes into `data`, the caller's inputs stay."""
        work, model = self._rectified(data, who)
        self._match_pairs(work, *self._backbone_pairs(work), static=static, capacity=capacity)
        live, ids = work.get("num_matches"), work["m_bids"]
        work["mkpts1_c"], _ = _map_back(data, model, work["mkpts1_c"], ids, live, inside=False)
        work["mkpts1_f"], work["minside1"] = _map_back(data, model, work["mkpts1_f"], ids, live)
        data.update({k: v for k, v in work.items() if k not in _INPUT_KEYS})

    def _match_searched(self, data, who, static=False, capacity=None):
        """forward / forward_static with data["rectify1_candidates"] (DESIGN.md §20), without a host sync beyond the
        eager call's one: image0's backbone once, the warped image1 of all N * K candidates, the coarse stage with the
        search (CoarseMatching.run), the fine stage over the winners' matches in candidate space; then pair ids and
        mkpts1_c / mkpts1_f mapped back through the chosen candidates.  The caller's inputs stay."""
        for key in ("rectify1", "guide"):
            if data.get(key) is not None:
                raise ValueError(f"{who}: data['rectify1_candidates'] cannot be combined with data['{key}']")
        img0 = data["image0"]
        cands = check_rectify_candidates(data["rectify1_candidates"], img0.shape[0], img0.device, who)
        n, k = cands.shape[:2]
        work = _warped_input(data, cands.view(n * k, 3, 3), k, who)
        (feat_c0, feat_f0), (feat_c1, feat_f1) = self._backbone(img0), self._backbone(work["image1"])
        work.update({"bs": n * k, "hw0_i": img0.shape[2:], "hw1_i": img0.shape[2:], "hw0_c": feat_c0.shape[2:],
                     "hw1_c": feat_c1.shape[2:], "hw0_f": feat_f0.shape[2:], "hw1_f": feat_f1.shape[2:]})
        cand = torch.arange(n * k, dtype=torch.int32, device=img0.device)   # candidate c = b * K + k reads image0[b]
        self._match_pairs(work, feat_c0, feat_c1, feat_f0, feat_f1, img_idx=(cand // k, cand), static=static,
                          capacity=capacity, search=k)
        pair = torch.arange(n, device=img0.device)
        chosen = cands[pair, work["rectify1_choice"]]
        work["b_ids"].div_(k, rounding_mode="floor")   # candidate ids -> pair ids
        if work["m_bids"] is not work["b_ids"]:   # a list of its own only when thr < 0
            work["m_bids"].div_(k, rounding_mode="floor")
        live, ids = work.get("num_matches"), work["m_bids"]
        work["mkpts1_c"], _ = _map_back(data, chosen, work["mkpts1_c"], ids, live, inside=False)
        work["mkpts1_f"], work["minside1"] = _map_back(data, chosen, work["mkpts1_f"], ids, live)
        if "conf_matrix" in work:
            work["conf_matrix"] = work["conf_matrix"].view(n, k, *work["conf_matrix"].shape[1:])[
                pair, work["rectify1_choice"]]
        work["bs"] = n
        data.update({key: v for key, v in work.items() if key not in _INPUT_KEYS})

    @torch.no_grad()
    def match_points(self, data, points0=None, valid0=None, *, points1=None, valid1=None, round_trip=False):
        """Refines caller-given image0 points to image1 through the coarse and fine stages (DESIGN.md §17).

        data: forward's inputs (image0 / image1, optional mask0 / mask1 and scale0 / scale1), all on the device.
        points0: float32 [N, Q, 2] (x, y) in image0 pixels, or in source pixels when scale0 is given (as mkpts0_f).
        valid0: optional bool [N, Q]; false marks a slot that is not a query.

        Writes qpts0_f (the query snapped to the fine grid), qpts1_c (centre of the image1 search window), qpts1_f (the
        refined correspondence), all [N, Q, 2] f32 in source pixels; qexpec_f [N, Q, 3] (as expec_f); qconf [N, Q]
        (mconf's expression for the chosen cell pair); q_i_ids / q_j_ids [N, Q] int64 (the query's cell and its best
        cell in image1, -1: none); qmutual, qvalid (the forward would keep the pair, before any per-pair cap) and
        qinside (the query was answered) [N, Q] bool.  A query that is not inside has NaN points and qexpec_f, qconf 0,
        false flags and ids -1.  Nothing of forward's match list is written.

        Each query's outputs depend only on its own point, pair and images.  A query at a forward match's mkpts0_c gets
        that match's j_ids, mconf, mkpts1_c, mkpts1_f and expec_f bit for bit.  Shapes are fixed by [N, Q] and there is
        no host synchronisation, so the call can be captured by `torch.cuda.graph` after one eager call.
        A guide (data["guide"]) is not supported here and raises ValueError.

        data["rectify1"] (as in `forward`): the queries are answered on the substituted input; qpts1_c / qpts1_f are
        mapped back into image1 and qinside1 [N, Q] bool says whether qpts1_f lies in image1's valid area; qexpec_f
        and q_j_ids stay in the rectified frame.

        points1 / valid1 (keyword-only, instead of points0 / valid0): image1 points, answered in image0 on the same
        coarse and fine evidence (DESIGN.md §22).  The keys follow "qptsX_* is in image X": qpts1_f (the snapped
        query), qpts0_c (the image0 window centre), qpts0_f (the answer), qexpec_f (in image0's window); q_i_ids /
        q_j_ids stay the image0 / image1 cells, i being the column arg-max of the query's cell j.  A query at a forward
        match's mkpts1_c gets that match's ids, mconf and flags bit for bit.

        round_trip: answer the first leg's answers back from the other image, with qinside as their validity, on the
        same coarse pass (no score pass runs again).  Adds qback_pts [N, Q, 2] (the back answer, in the query's own
        image), qback_conf, qback_valid, qback_inside [N, Q] (as qconf, qvalid, qinside for the back leg) and qfb_err
        [N, Q] f32 (|qback_pts - the query| in source pixels, NaN unless both legs are inside).  The back leg equals a
        call from the other image with points = the first answer and valid = qinside, bit for bit.
        Neither points1 nor round_trip combines with data["rectify1"]."""
        _require_eval(self)
        side, points, valid = _query_side(points0, valid0, points1, valid1, round_trip, "match_points")
        if data.get("guide") is not None:
            raise ValueError("match_points: data['guide'] is not supported (guided matching is available in forward, "
                             "forward_static and match_features)")
        if data.get("rectify1_candidates") is not None:
            raise ValueError("match_points: data['rectify1_candidates'] is not supported (the rectification search is "
                             "available in forward and forward_static; pass the chosen model as data['rectify1'])")
        _lib.require_entries(_lib.POINTS_ENTRIES, "match_points")
        if side or round_trip:
            _lib.require_entries(_lib.SIDE_POINTS_ENTRIES, "match_points")
        _check_points(data, points, valid, side)
        if data.get("rectify1") is None:
            self._match_points(data, points, valid, side=side, round_trip=round_trip)
            return
        if side or round_trip:
            raise ValueError("match_points: points1 and round_trip cannot be combined with data['rectify1']")
        work, model = self._rectified(data, "match_points")
        self._match_points(work, points0, valid0)
        n, q = points0.shape[:2]
        ids = torch.arange(n, device=points0.device)[:, None].expand(n, q).reshape(-1)   # query b*Q + k is of pair b
        work["qpts1_c"] = _map_back(data, model, work["qpts1_c"].view(-1, 2), ids, inside=False)[0].view(n, q, 2)
        pts, inside = _map_back(data, model, work["qpts1_f"].view(-1, 2), ids)
        work["qpts1_f"], work["qinside1"] = pts.view(n, q, 2), inside.view(n, q)
        data.update({k: v for k, v in work.items() if k not in _INPUT_KEYS})

    def _match_points(self, data, points, valid, feats=None, img_idx=None, side=0, round_trip=False):
        """match_points / match_points_features on validated arguments: `points` / `valid` of image `side`.
        feats: None (the backbone runs on data's image0 / image1), or the (feat_c0, feat_c1, feat_f0, feat_f1) banks of
        a pair list, read at img_idx = (idx0, idx1) as in `_match_pairs`; `data` then already holds bs and the sizes.
        round_trip: the back leg runs on the coarse workspace of the first (DESIGN.md §22)."""
        n, q = points.shape[:2]
        dev = points.device
        if q == 0:
            data.update(_query_outputs(n, 0, dev, side, round_trip))
            return
        feat_c0, feat_c1, feat_f0, feat_f1 = self._backbone_pairs(data) if feats is None else feats
        c = feat_c0.shape[1]
        (h0, w0), (h1, w1) = data["hw0_c"], data["hw1_c"]
        L, S = h0 * w0, h1 * w1
        state, m0, m1 = self._coarse_tokens(data, feat_c0, feat_c1, img_idx)
        coarse = (state.cat_hi, state.cat_lo, 2 * c, n, L, S, c, data, m0, m1)
        ws = None
        if round_trip:
            ws = torch.empty(_lib.load().lb_coarse_match_workspace_bytes(n, L, S), dtype=torch.uint8, device=dev)
        fine = (feat_f0.float(), feat_f1.float(), state.x, n, L, S, data, img_idx)
        out = self.coarse_matching.query(*coarse, points, valid, side=side, ws=ws)
        self._fine_points(out, side, *fine)
        if round_trip:
            other = 1 - side
            back = self.coarse_matching.query(*coarse, out[f"qpts{other}_f"], out["qinside"], side=other, ws=ws,
                                              reuse=True)
            self._fine_points(back, other, *fine)
            pts, inside = back[f"qpts{side}_f"], back["qinside"]
            err = torch.linalg.vector_norm(pts - points, dim=-1)
            out.update({"qback_pts": pts, "qback_conf": back["qconf"], "qback_valid": back["qvalid"],
                        "qback_inside": inside, "qfb_err": err.masked_fill_(~inside, float("nan"))})
        data.update(out)

    def _fine_points(self, out, side, feat_f0, feat_f1, x, n, L, S, data, img_idx):
        """The fine stage of the queries of CoarseMatching.query's `out` (image `side`), in place: pops its centres and
        window ids and adds the answer qpts{1 - side}_f and qexpec_f.  The fine state is freed on return."""
        q = out["qinside"].shape[1]
        centres, win = out.pop("centres"), out.pop("win_ids")
        inside = out["qinside"].reshape(-1)
        # the fine stage reads the windows as a match list of N*Q entries: (b, i, j) = win_ids
        work = {k: data[k] for k in ("bs", "hw0_i", "hw1_i", "hw0_c", "hw1_c", "hw0_f", "hw1_f", "scale0", "scale1")
                if k in data}
        work.update({"b_ids": win[0], "i_ids": win[1], "j_ids": win[2]})
        fstate = self.fine_preprocess.run(feat_f0, feat_f1, x, n, L, S, work, img_idx=img_idx,
                                          centres=(centres, inside))
        ww = self.fine_preprocess.W ** 2
        self.loftr_fine.run(fstate, n * q, ww, ww)
        f0, f1 = fstate.sides(n * q, ww, ww)
        if side == 0:
            work.update({"mkpts0_c": out["qpts0_f"].view(-1, 2), "mkpts1_c": out["qpts1_c"].view(-1, 2)})
            self.fine_matching(f0, f1, work)
        else:   # the mirror: window1's centre against window0, refined from the image0 centre with scale0
            if "scale0" in work:
                work["scale0"], work["scale1"] = work["scale1"], work["scale0"]
            work.update({"mkpts0_c": out["qpts1_f"].view(-1, 2), "mkpts1_c": out["qpts0_c"].view(-1, 2)})
            self.fine_matching(f1, f0, work)
        out[f"qpts{1 - side}_f"] = work["mkpts1_f"].view(n, q, 2)
        out["qexpec_f"] = work["expec_f"].view(n, q, 3).masked_fill_(~out["qinside"][..., None], float("nan"))

    def _backbone_pairs(self, data):
        """Step 1 of the forward (no host sync): the backbone on image0 / image1 -> (feat_c0, feat_c1, feat_f0,
        feat_f1); writes bs and the image, coarse and fine sizes into `data`."""
        img0, img1 = data["image0"], data["image1"]
        bs = img0.size(0)
        data.update({"bs": bs, "hw0_i": img0.shape[2:], "hw1_i": img1.shape[2:]})

        # 1. local feature CNN                                                         [loftr.py:45-49]
        if data["hw0_i"] == data["hw1_i"]:
            feats_c, feats_f = self._backbone(torch.cat([img0, img1], dim=0))
            (feat_c0, feat_c1), (feat_f0, feat_f1) = feats_c.split(bs), feats_f.split(bs)
        else:
            (feat_c0, feat_f0), (feat_c1, feat_f1) = self._backbone(img0), self._backbone(img1)
        data.update({"hw0_c": feat_c0.shape[2:], "hw1_c": feat_c1.shape[2:],
                     "hw0_f": feat_f0.shape[2:], "hw1_f": feat_f1.shape[2:]})
        return feat_c0, feat_c1, feat_f0, feat_f1

    def _match_pairs(self, data, feat_c0, feat_c1, feat_f0, feat_f1, img_idx=None, static=False, capacity=None,
                     search=None):
        """Steps 2-5 of the forward for the data["bs"] pairs whose sizes `data` holds: position encoding and token
        layout, coarse transformer, coarse matching, fine preprocess and transformer, fine matching.
        img_idx: optional (idx0, idx1) int32 [bs]: the maps are then feature banks, read at image idx0[b] / idx1[b] for
        pair b.  static: the match keys are buffers of `capacity` entries (None: the default capacity) and the fine
        stage is bounded on the device by their count (CoarseMatching.run), so that nothing synchronises with the host.
        search: None, or K: the bs pairs are candidates of a rectification search (CoarseMatching.run)."""
        bs, c = data["bs"], feat_c0.shape[1]
        (h0, w0), (h1, w1) = data["hw0_c"], data["hw1_c"]
        L, S = h0 * w0, h1 * w1
        state, m0, m1 = self._coarse_tokens(data, feat_c0, feat_c1, img_idx)

        # 3. coarse matching                                                           [loftr.py:67]
        live = self.coarse_matching.run(state.cat_hi, state.cat_lo, 2 * c, bs, L, S, c, data, m0, m1, static, capacity,
                                        search)

        # 4. fine-level refinement over M windows: the match count, or the capacity    [loftr.py:70-72]
        fstate = self.fine_preprocess.run(feat_f0.float(), feat_f1.float(), state.x, bs, L, S, data, live, img_idx)
        m, ww = data["b_ids"].shape[0], self.fine_preprocess.W ** 2
        if m:
            self.loftr_fine.run(fstate, m, ww, ww, live=live)

        # 5. fine matching                                                             [loftr.py:75]
        self.fine_matching(*fstate.sides(m, ww, ww), data, live=live)
        if self.expose_coarse_features:   # test / debugging tap, off by default: not a reference key
            data["_feat_c0"], data["_feat_c1"] = state.sides(bs, L, S)

    def _coarse_tokens(self, data, feat_c0, feat_c1, img_idx=None):
        """Step 2 of the forward: position encoding, token layout and coarse transformer (img_idx as in
        `_match_pairs`) -> (token state, flattened uint8 mask0, mask1 views or None)."""
        # 2. position encoding + token layout + coarse transformer                     [loftr.py:58-64]
        lib = _lib.load()
        bs = data["bs"]
        nhwc = self._tc_backbone is not None
        c = feat_c0.shape[1]
        (h0, w0), (h1, w1) = data["hw0_c"], data["hw1_c"]
        L, S = h0 * w0, h1 * w1
        state = _TokenState(bs * L, bs * S, c, feat_c0.device)
        pe = self.pos_encoding.pe[0]
        st = _stream(feat_c0)
        idx0, idx1 = (None, None) if img_idx is None else img_idx
        for feat, idx, h, w, row0 in ((feat_c0, idx0, h0, w0, 0), (feat_c1, idx1, h1, w1, bs * L)):
            feat = feat.float()
            feat = feat.permute(0, 2, 3, 1).contiguous() if nhwc else feat.contiguous()   # no copy in either case
            out = (state.x.data_ptr() + row0 * c * 4, state.cat_hi.data_ptr() + row0 * 2 * c * 2,
                   state.cat_lo.data_ptr() + row0 * 2 * c * 2, st)
            if idx is None:
                _lib.check(lib.lb_coarse_prep(feat.data_ptr(), int(nhwc), pe.data_ptr(), bs, c, h, w, pe.shape[1],
                                              pe.shape[2], *out))
            else:
                _lib.check(lib.lb_coarse_prep_indexed(feat.data_ptr(), int(nhwc), pe.data_ptr(), idx.data_ptr(), bs, c,
                                                      h, w, pe.shape[1], pe.shape[2], *out))
        mask_all = m0 = m1 = None
        if "mask0" in data:
            m0 = data["mask0"].flatten(-2).reshape(-1).to(torch.uint8)
            m1 = data["mask1"].flatten(-2).reshape(-1).to(torch.uint8)
            mask_all = torch.cat([m0, m1]).contiguous()
            m0, m1 = mask_all[: bs * L], mask_all[bs * L:]
        self.loftr_coarse.run(state, bs, L, S, mask_all)
        return state, m0, m1

    def _packed_caches(self):
        """Every owner of a packed-weight cache: the caching submodules and the tensor-core backbone."""
        caches = [m for m in self.modules() if isinstance(m, _PackedCache)]
        return caches if self._tc_backbone is None else caches + [self._tc_backbone]

    def invalidate_packed(self):
        """Drop every packed-weight cache (fp16 hi/lo planes, folded BatchNorm): required after parameter writes
        that PyTorch cannot see (`.data` mutation); implied by load_state_dict / .to() / .cuda() / .float()."""
        for m in self._packed_caches():
            m.invalidate_packed()

    def _apply(self, fn, *args, **kwargs):
        self.invalidate_packed()
        return super()._apply(fn, *args, **kwargs)

    def load_state_dict(self, state_dict, *args, **kwargs):
        """Accepts checkpoints saved from the Lightning wrapper ('matcher.' prefix; reference loftr.py:77-81)."""
        for k in list(state_dict.keys()):
            if k.startswith("matcher."):
                state_dict[k.replace("matcher.", "", 1)] = state_dict.pop(k)
        self.invalidate_packed()
        return super().load_state_dict(state_dict, *args, **kwargs)


# forward's inputs: a rectified call copies every other key of its work dict back to the caller's
_INPUT_KEYS = ("image0", "image1", "mask0", "mask1", "scale0", "scale1")


def _require_static(model, capacity, what):
    """Preconditions of the sync-free forward (`what`: the public entry point), checked before any launch."""
    _require_eval(model)
    if model.coarse_matching.thr < 0:
        raise ValueError(f"{what} needs match_coarse.thr >= 0: with thr < 0 the reference's mconf != 0 filter makes "
                         "the output list depend on the data")
    if capacity is not None and int(capacity) < 1:
        raise ValueError(f"capacity must be a positive number of matches (got {capacity})")


_QUERY_KEYS = {"qpts0_f": (torch.float32, 2), "qpts1_c": (torch.float32, 2), "qpts1_f": (torch.float32, 2),
               "qexpec_f": (torch.float32, 3), "qconf": (torch.float32, 0), "q_i_ids": (torch.int64, 0),
               "q_j_ids": (torch.int64, 0), "qmutual": (torch.bool, 0), "qvalid": (torch.bool, 0),
               "qinside": (torch.bool, 0)}


# the round trip's keys (DESIGN.md §22)
_BACK_KEYS = {"qback_pts": (torch.float32, 2), "qback_conf": (torch.float32, 0), "qback_valid": (torch.bool, 0),
              "qback_inside": (torch.bool, 0), "qfb_err": (torch.float32, 0)}


def _query_outputs(n, q, dev, side=0, round_trip=False):
    """Empty output tensors of LoFTR.match_points for [n, q] queries of image `side` (qptsX_* keys in image X)."""
    keys = {k.translate(str.maketrans("01", "10")) if side and k.startswith("qpts") else k: v
            for k, v in _QUERY_KEYS.items()}
    if round_trip:
        keys.update(_BACK_KEYS)
    return {k: torch.empty(n, q, *((d,) if d else ()), dtype=t, device=dev) for k, (t, d) in keys.items()}


def _query_side(points0, valid0, points1, valid1, round_trip, who):
    """The queried image of a match_points / match_points_features call (`who`) -> (side, points, valid).  Without
    points1 the points0 checks run as before, so a call that gives neither fails on points0."""
    if not isinstance(round_trip, bool):
        raise TypeError(f"{who}: round_trip must be a bool (got {type(round_trip).__name__})")
    if points1 is None:
        if valid1 is not None:
            raise ValueError(f"{who}: valid1 is given without points1")
        return 0, points0, valid0
    if points0 is not None or valid0 is not None:
        raise ValueError(f"{who}: give the queries of one image: points0 (and valid0) or points1 (and valid1)")
    return 1, points1, valid1


def _check_points(data, points0, valid0, side=0):
    """Host-side validation of LoFTR.match_points' arguments, before any launch: shapes and dtypes first, then that
    everything is on image0's CUDA device."""
    for k in ("image0", "image1"):
        if k not in data:
            raise ValueError(f"match_points: data must hold `{k}`")
    check_pairs(data["image0"].shape[0], "match_points")
    if ("scale0" in data) != ("scale1" in data):
        raise ValueError("match_points: give scale0 and scale1 together")
    if ("mask0" in data) != ("mask1" in data):
        raise ValueError("match_points: give mask0 and mask1 together")
    _check_query_args(points0, valid0, data["image0"].shape[0], "match_points", side)
    named = [(k, data[k]) for k in ("image0", "image1", "mask0", "mask1", "scale0", "scale1") if k in data]
    _check_devices(named + [(f"points{side}", points0)] + ([(f"valid{side}", valid0)] if valid0 is not None else []),
                   data["image0"].device, "image0", "match_points")


def _check_query_args(points0, valid0, n, who, side=0):
    """Dtypes and shapes of the queries of `n` pairs (match_points / match_points_features, `who`); the messages name
    points{side} / valid{side}."""
    p, v = f"points{side}", f"valid{side}"
    if not torch.is_tensor(points0) or points0.dtype != torch.float32:
        raise TypeError(f"{who}: {p} must be a float32 tensor (got "
                        f"{points0.dtype if torch.is_tensor(points0) else type(points0).__name__})")
    if points0.dim() != 3 or points0.shape[0] != n or points0.shape[2] != 2:
        raise ValueError(f"{who}: {p} must be [N, Q, 2] with N = {n} pairs (got {tuple(points0.shape)})")
    if valid0 is not None:
        if not torch.is_tensor(valid0) or valid0.dtype != torch.bool:
            raise TypeError(f"{who}: {v} must be a bool tensor")
        if tuple(valid0.shape) != tuple(points0.shape[:2]):
            raise ValueError(f"{who}: {v} must be [N, Q] = {tuple(points0.shape[:2])} (got {tuple(valid0.shape)})")


def _check_devices(named, dev, what, who):
    """Every (name, tensor) of `named` is a CUDA tensor on `dev`, the device of `what`."""
    for k, t in named:
        if not torch.is_tensor(t) or not t.is_cuda:
            raise ValueError(f"{who}: `{k}` must be a CUDA tensor")
        if t.device != dev:
            raise ValueError(f"{who}: `{k}` is on {t.device}, {what} on {dev}")


def _bank_sizes(bs, feats0, feats1):
    """The bookkeeping keys forward writes (bs and the image, coarse and fine sizes) for `bs` pairs of two banks."""
    return {"bs": bs, "hw0_i": feats0.hw_i, "hw1_i": feats1.hw_i, "hw0_c": feats0.hw_c, "hw1_c": feats1.hw_c,
            "hw0_f": feats0.hw_f, "hw1_f": feats1.hw_f}


def _bank_inputs(feats0, idx0, feats1, idx1, scale0, scale1, dev, who, gather=True):
    """forward's per-pair masks and scales of a checked pair list (LoFTR._check_banks), gathered through the indices
    -> dict with mask0 / mask1 and scale0 / scale1 where given.  The scale shapes are checked before the gathers;
    gather=False checks them only (an empty dict, nothing launched)."""
    if scale0 is not None:
        for name, s, f in (("scale0", scale0, feats0), ("scale1", scale1, feats1)):
            if tuple(s.shape) != (len(f), 2):
                raise ValueError(f"{who}: {name} must be [{len(f)}, 2] (got {tuple(s.shape)})")
    work = {}
    if not gather:
        return work
    if feats0.mask is not None:
        work["mask0"], work["mask1"] = feats0.mask[idx0.long()], feats1.mask[idx1.long()]
    if scale0 is not None:
        work["scale0"], work["scale1"] = scale0.to(dev)[idx0.long()], scale1.to(dev)[idx1.long()]
    return work


def _weight_refs(model):
    """(packed-weight cache objects, parameters + buffers, their (data_ptr, _version) key) of `model`: everything a
    captured graph holds raw device pointers into."""
    caches = [m._packed for m in model._packed_caches()]
    return caches, list(model.parameters()) + list(model.buffers()), _weights_key(model)


class ImageFeatures:
    """Backbone output of K images of one size (`LoFTR.extract_features`), matched pair by pair with
    `LoFTR.match_features` without running the backbone again.

    feat_c [K, C_c, H/8, W/8] and feat_f [K, C_f, H/2, W/2] are the maps as the backbone emits them (NHWC storage,
    i.e. channels-last strides, from the tensor-core backbone; NCHW from the PyTorch one); mask: optional padding
    masks [K, H/8, W/8]; hw_i / hw_c / hw_f: image, coarse and fine sizes.  weights_key identifies the backbone weights the
    bank was extracted with."""

    def __init__(self, feat_c, feat_f, mask, hw_i, hw_c, hw_f, weights_key):
        self.feat_c, self.feat_f, self.mask = feat_c, feat_f, mask
        self.hw_i, self.hw_c, self.hw_f = hw_i, hw_c, hw_f
        self.weights_key = weights_key

    def __len__(self):
        return self.feat_c.shape[0]


class CapturedMatcher:
    """`model(data)` replayed from one CUDA graph: a drop-in for the matcher call in a loop over fixed-size batches
    (video, SLAM front ends, webcam demos), where the host cost of enqueueing every launch would otherwise be paid per
    frame.

    The constructor allocates static input buffers for `batch` pairs of `hw0` / `hw1` images (plus masks and scales
    when asked for), runs one eager `model.forward_static` to warm up (weight packing, kernel attributes, cuDNN
    algorithm selection) and captures the next one.  `__call__(data)` copies the inputs into the static buffers,
    replays the graph and reads the match count once (the only host sync); it fills `data` with the same keys, shapes
    and values as `model(data)`.  The trimmed outputs are copies, valid after later replays.

    The graph holds raw pointers into the model's packed-weight caches, parameters and buffers.  The captured matcher
    keeps those objects alive and, on every call, checks on the host that the model still uses them: after
    `load_state_dict`, `.to()`, `invalidate_packed()` or a parameter change a call raises instead of replaying against
    stale weights; `recapture()` rebuilds the graph.  The same holds for `model.coarse_matching.max_matches_per_pair`,
    which is captured with the graph.  See `LoFTR.forward_static` for `capacity` and its memory cost."""

    _TRIMMED = ("b_ids", "i_ids", "j_ids", "gt_mask", "mconf", "mkpts0_c", "mkpts1_c", "mkpts1_f", "expec_f")

    def __init__(self, model, batch, hw0, hw1=None, masks=False, scales=False, capacity=None):
        _require_static(model, capacity, "CapturedMatcher")
        dev = next(model.parameters()).device
        if dev.type != "cuda":
            raise ValueError("CapturedMatcher: the model must live on a CUDA (H100) device; call .cuda() first")
        hw1 = hw0 if hw1 is None else hw1
        (h0, w0), (h1, w1) = hw0, hw1
        res = model.config["resolution"][0]
        self.model, self.device, self.capacity_arg = model, dev, capacity
        self.static = {"image0": torch.zeros(batch, 1, h0, w0, device=dev),
                       "image1": torch.zeros(batch, 1, h1, w1, device=dev)}
        if masks:
            self.static["mask0"] = torch.ones(batch, h0 // res, w0 // res, dtype=torch.bool, device=dev)
            self.static["mask1"] = torch.ones(batch, h1 // res, w1 // res, dtype=torch.bool, device=dev)
        if scales:
            self.static["scale0"] = torch.ones(batch, 2, device=dev)
            self.static["scale1"] = torch.ones(batch, 2, device=dev)
        self.graph = None
        self.recapture()

    @property
    def capacity(self):
        return int(self.out["b_ids"].shape[0])

    def recapture(self):
        """(Re)runs the eager warm-up and captures a new graph against the model's current weights."""
        self.graph = self.out = self._refs = None
        max_per_pair = self.model.coarse_matching.max_matches_per_pair
        with torch.cuda.device(self.device):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self.model.forward_static(dict(self.static), self.capacity_arg)
            torch.cuda.current_stream().wait_stream(side)
            graph, out = torch.cuda.CUDAGraph(), dict(self.static)
            with torch.cuda.graph(graph):
                self.model.forward_static(out, self.capacity_arg)
        self.graph, self.out, self._refs = graph, out, _weight_refs(self.model)
        self.max_matches_per_pair = max_per_pair

    def _check_weights(self):
        caches, tensors, key = _weight_refs(self.model)
        c0, t0, k0 = self._refs
        if len(caches) != len(c0) or any(a is not b for a, b in zip(caches, c0)) or len(tensors) != len(t0) or \
                any(a is not b for a, b in zip(tensors, t0)) or key != k0:
            raise RuntimeError("loftr_b200.CapturedMatcher: weights changed since capture (load_state_dict, .to(), "
                               "invalidate_packed() or a parameter update); call recapture()")

    def __call__(self, data):
        for k, what in (("guide", "a guide"), ("rectify1", "rectify1"), ("rectify1_candidates", "rectify1_candidates")):
            if data.get(k) is not None:
                raise ValueError(f"CapturedMatcher: data['{k}'] is not supported (capture LoFTR.forward_static with "
                                 f"{what} instead)")
        if self.graph is None:
            raise RuntimeError("loftr_b200.CapturedMatcher: no captured graph; call recapture()")
        self._check_weights()
        now = self.model.coarse_matching.max_matches_per_pair
        if now != self.max_matches_per_pair:
            raise RuntimeError(f"loftr_b200.CapturedMatcher: coarse_matching.max_matches_per_pair changed since capture "
                               f"({self.max_matches_per_pair} -> {now}); call recapture()")
        for k, buf in self.static.items():
            if k not in data:
                raise ValueError(f"CapturedMatcher was built with `{k}` but the call does not provide it")
            if tuple(data[k].shape) != tuple(buf.shape):
                raise ValueError(f"CapturedMatcher: `{k}` has shape {tuple(data[k].shape)}, captured {tuple(buf.shape)}")
        for k in ("mask0", "mask1", "scale0", "scale1"):
            if k in data and k not in self.static:
                raise ValueError(f"CapturedMatcher was built without `{k}`; construct it with masks=/scales=True")
        with torch.cuda.device(self.device):
            for k, buf in self.static.items():
                buf.copy_(data[k])
            self.graph.replay()
            m = int(self.out["num_matches"].item())   # the one host sync
        if m > self.capacity:
            raise RuntimeError(f"loftr_b200.CapturedMatcher: {m} coarse matches exceed the capacity {self.capacity}; "
                               "construct it with a larger capacity")
        res = {}
        for k, v in self.out.items():
            if k in self.static or k in ("num_matches", "m_bids", "mkpts0_f"):
                continue
            if k in self._TRIMMED:
                res[k] = v[:m].clone()
            elif torch.is_tensor(v):
                res[k] = v.clone()
            else:
                res[k] = v
        res["m_bids"], res["mkpts0_f"] = res["b_ids"], res["mkpts0_c"]   # aliased as in `forward`
        data.update(res)
