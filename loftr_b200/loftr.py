"""`LoFTR(config)` / `matcher(batch)` -- the drop-in boundary (reference src/loftr/loftr.py:12-81).

Same constructor argument (the lower-case config dict), same sub-module and parameter names (so
`state_dict`s and released checkpoints round-trip), same `forward(data) -> None` contract that
mutates `data` with the reference's output keys.  Everything runs in the hand-written sm_90a kernels behind the
C ABI of include/loftr_b200.h: the ResNet-FPN backbone as implicit-GEMM convolutions on the tensor cores
(`backbone_impl="b200"`, the default for the shipped ResNetFPN_8_2 shape; `"torch"` keeps the PyTorch/cuDNN fp32
forward, which is closer to fp64 -- DESIGN.md §10), then position encoding, coarse transformer, coarse
matching, fine windows, fine transformer and fine matching.
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

import torch
import torch.nn as nn

from . import _lib
from .backbone import build_backbone

_KIND = {("self", "linear"): _lib.LAYER_SELF, ("cross", "linear"): _lib.LAYER_CROSS,
         ("self", "full"): _lib.LAYER_SELF_FULL, ("cross", "full"): _lib.LAYER_CROSS_FULL}
ATTENTIONS = ("linear", "full")   # reference config: coarse.attention / fine.attention, options ['linear', 'full']


def _stream(ref=None):
    """cudaStream_t of torch's current stream ON THE DEVICE THAT OWNS `ref` (a tensor or torch.device); the library
    binds itself to the device of the buffers it is given, so the stream handle must belong to that device too."""
    dev = ref.device if torch.is_tensor(ref) else ref
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


class _PackedCacheMixin:
    """Keeps the ctypes / device-plane weight caches out of deepcopy / pickle state and drops them whenever the
    parameters are re-materialised (`_apply`: .to / .cuda / .float / .half) or re-loaded."""
    _CACHE_ATTRS = ("_packed", "_packed_key")

    def invalidate_packed(self):
        for a in self._CACHE_ATTRS:
            if a in self.__dict__:
                self.__dict__[a] = None

    def __getstate__(self):
        d = dict(self.__dict__)
        for a in self._CACHE_ATTRS:
            if a in d:
                d[a] = None
        return d

    def _apply(self, fn, *args, **kwargs):
        self.invalidate_packed()
        return super()._apply(fn, *args, **kwargs)

    def _load_from_state_dict(self, *args, **kwargs):
        self.invalidate_packed()
        return super()._load_from_state_dict(*args, **kwargs)


def _require_cuda(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"loftr_b200: `{name}` must live on a CUDA (H100) device; the matching hot path has "
                           "no CPU implementation")


def split_weight(w: torch.Tensor):
    """Weight matrix -> (hi, lo, acc_scale): planes of w * 2^e with e chosen so that max|w| * 2^e ~ 2^12, and
    acc_scale = 2^-e for the epilogue.  Power-of-two scaling is exact; it moves the `lo` residuals of typical
    (small) weights out of fp16's subnormal range, where they would only carry ~1e-6 relative accuracy."""
    w = w.detach().float().contiguous()
    amax = float(w.abs().max())
    e = 0 if amax == 0.0 else int(math.floor(math.log2(4096.0 / amax)))
    e = max(min(e, 24), -24)
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


class TensorCoreBackbone:
    """ResNetFPN_8_2 forward through `lb_backbone_forward` (implicit-GEMM convolutions on wgmma).  Holds no
    parameters of its own: it packs the weights of the PyTorch `ResNetFPN` module it wraps (BatchNorm folded
    with its running statistics = eval mode), lazily and again whenever a parameter or buffer changes."""

    def __init__(self, torch_backbone):
        self.m = torch_backbone
        self._packed = None
        self._key = None

    def invalidate_packed(self):
        self._packed = None
        self._key = None

    def __getstate__(self):   # the cache holds ctypes structures with device pointers: never copied / pickled
        return {"m": self.m, "_packed": None, "_key": None}

    @staticmethod
    def supported(torch_backbone) -> bool:
        m = torch_backbone
        return getattr(m, "depth", 0) == 3 and m.conv1.out_channels == 128 and m.layer1[0].conv1.out_channels == 128 \
            and max(m.layer2[0].conv1.out_channels, m.layer3[0].conv1.out_channels) <= 256

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
        hi, lo, acc_scale = split_weight(torch.cat(planes, 1))
        nmain = k * k * cmain
        hi_m, lo_m = hi[:, :nmain].contiguous(), lo[:, :nmain].contiguous()
        hi_r = lo_r = None
        if rem.value:
            hi_r, lo_r = hi[:, nmain:].contiguous(), lo[:, nmain:].contiguous()
        scale, shift = self._fold(bn, cout, w.device)
        scale = (scale * acc_scale).contiguous()   # y = acc * (2^-e * bn_scale) + bn_shift
        keep += [hi_m, lo_m, hi_r, lo_r, scale, shift]
        return _lib.LbConvWeights(hi_m.data_ptr(), lo_m.data_ptr(), _lib.ptr(hi_r), _lib.ptr(lo_r), scale.data_ptr(),
                                  shift.data_ptr(), cin, cout, k, conv.stride[0])

    def _pack(self):
        m = self.m
        tensors = list(m.parameters()) + list(m.buffers())
        key = tuple(t._version for t in tensors) + tuple(t.data_ptr() for t in tensors)
        if self._packed is not None and self._key == key:
            return self._packed
        keep = []
        w = _lib.LbBackboneWeights()
        with torch.no_grad():
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
        self._packed, self._key = (w, keep), key
        return self._packed

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
        nbytes = lib.lb_backbone_workspace_bytes(C.byref(w), n, h, wd)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=images.device)
        _lib.check(lib.lb_backbone_forward(C.byref(w), images.data_ptr(), n, h, wd, feat_c.data_ptr(),
                                           feat_f.data_ptr(), ws.data_ptr(), nbytes, _stream(images)))
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


class LocalFeatureTransformer(_PackedCacheMixin, nn.Module):
    """Interleaved self/cross encoder with linear or full (softmax) attention (reference transformer.py:61-101)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.d_model = config["d_model"]
        self.nhead = config["nhead"]
        self.layer_names = list(config["layer_names"])
        self.layers = nn.ModuleList([LoFTREncoderLayer(config["d_model"], config["nhead"], config["attention"])
                                     for _ in self.layer_names])
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        self._packed = None
        self._packed_key = None

    # -- weight packing: fp16 hi/lo planes of the [out, in] matrices, built lazily per device/version
    def _pack(self, device):
        key = (str(device),) + tuple(p._version for p in self.parameters()) + tuple(p.data_ptr() for p in self.parameters())
        if self._packed is not None and self._packed_key == key:
            return self._packed
        keep = []
        arr = (_lib.LbEncoderLayerWeights * len(self.layers))()
        with torch.no_grad():
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
        self._packed = (arr, kinds, keep)
        self._packed_key = key
        return self._packed

    def run(self, state: _TokenState, n_groups, group_rows0, group_rows1, mask_u8=None, live=None):
        """In-place transformer over a prepared token state (used by LoFTR.forward).  `live` (fine windows only): an
        int32 device count; `n_groups` is then the capacity and only the first min(live, n_groups) windows of each set
        are computed."""
        lib = _lib.load()
        if any(layer.attention == "full" for layer in self.layers):
            _lib.require_full_attention(lib)   # an older library would reject the layer kinds at the first launch
        arr, kinds, _ = self._pack(state.x.device)
        st = _lib.LbTransformerState(state.x.data_ptr(), state.cat_hi.data_ptr(), state.cat_lo.data_ptr(),
                                     _lib.ptr(mask_u8), n_groups, group_rows0, group_rows1, _lib.ptr(live))
        nbytes = lib.lb_transformer_workspace_bytes(self.d_model, self.nhead, n_groups, group_rows0, group_rows1)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=state.x.device)
        _lib.check(lib.lb_transformer_forward(arr, kinds, len(self.layers), self.d_model, self.nhead, C.byref(st),
                                              ws.data_ptr(), nbytes, _stream(state.x)))

    @torch.no_grad()
    def forward(self, feat0, feat1, mask0=None, mask1=None):
        """feat0 [N, L, C], feat1 [N, S, C] (+ optional bool masks [N, L], [N, S]) -> updated features."""
        assert self.d_model == feat0.size(2), "the feature number of src and transformer must be equal"
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
    (reference coarse_matching.py:59-261, eval path)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
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

    @staticmethod
    def default_capacity(n, L, S, masked):
        """Exact bound on the number of coarse matches: mutual nearest neighbours pair each row with at most one
        column, so n*min(L, S) without masks (n*L with masks, as padding may leave columns unmatched)."""
        return max(n * min(L, S) if not masked else n * L, 1)

    def run(self, hi, lo, ld, n, L, S, c, data, mask_u8_0=None, mask_u8_1=None):
        """Planes of feat_c0 (rows [0, n*L)) / feat_c1 (rows [n*L, ...)) -> coarse match keys in `data`."""
        cap = self.default_capacity(n, L, S, mask_u8_0 is not None)
        b_ids, i_ids, j_ids, mconf, mk0, mk1, count, conf = self._launch(hi, lo, ld, n, L, S, c, data, mask_u8_0,
                                                                         mask_u8_1, cap)
        dev = hi.device
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

    def run_static(self, hi, lo, ld, n, L, S, c, data, mask_u8_0, mask_u8_1, cap):
        """`run` without the host sync: the match keys of `data` are the fixed-capacity buffers ([cap] first
        dimension; entries at or past min(count, cap) unspecified) and the returned int32 device tensor [1] holds the
        true count.  Requires thr >= 0 (the `mconf != 0` filter of thr < 0 would be a second, data-dependent list)."""
        if self.thr < 0:
            raise ValueError("forward_static needs match_coarse.thr >= 0: with thr < 0 the mconf != 0 filter makes the "
                             "output list depend on the data")
        b_ids, i_ids, j_ids, mconf, mk0, mk1, count, conf = self._launch(hi, lo, ld, n, L, S, c, data, mask_u8_0,
                                                                         mask_u8_1, cap)
        data.update({"b_ids": b_ids, "i_ids": i_ids, "j_ids": j_ids,
                     "gt_mask": torch.zeros(cap, dtype=torch.bool, device=hi.device), "m_bids": b_ids,
                     "mkpts0_c": mk0, "mkpts1_c": mk1, "mconf": mconf, "num_matches": count})
        if conf is not None:
            data["conf_matrix"] = conf
        return count

    def _launch(self, hi, lo, ld, n, L, S, c, data, mask_u8_0, mask_u8_1, cap):
        """Enqueues lb_coarse_match into buffers of `cap` entries -> (b_ids, i_ids, j_ids, mconf, mkpts0_c, mkpts1_c,
        count, conf_matrix or None); no host sync."""
        if self.training:
            raise NotImplementedError("loftr_b200 builds the inference path only (no training-time sampling)")
        lib = _lib.load()
        dev = hi.device
        b_ids = torch.empty(cap, dtype=torch.int64, device=dev)
        i_ids = torch.empty(cap, dtype=torch.int64, device=dev)
        j_ids = torch.empty(cap, dtype=torch.int64, device=dev)
        mconf = torch.empty(cap, dtype=torch.float32, device=dev)
        mk0 = torch.empty(cap, 2, dtype=torch.float32, device=dev)
        mk1 = torch.empty(cap, 2, dtype=torch.float32, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
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
        a.capacity = cap
        a.b_ids, a.i_ids, a.j_ids = b_ids.data_ptr(), i_ids.data_ptr(), j_ids.data_ptr()
        a.mconf, a.mkpts0_c, a.mkpts1_c, a.count = mconf.data_ptr(), mk0.data_ptr(), mk1.data_ptr(), count.data_ptr()
        conf = None
        if self.config.get("return_conf_matrix", False):   # opt-in: 4*L*S bytes per pair, training-loss input only
            conf = torch.empty(n, L, S, dtype=torch.float32, device=dev)
            a.conf_matrix = conf.data_ptr()
        nbytes = lib.lb_coarse_match_workspace_bytes(n, L, S)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(lib.lb_coarse_match(C.byref(a), ws.data_ptr(), nbytes, _stream(hi)))
        return b_ids, i_ids, j_ids, mconf, mk0, mk1, count, conf

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


class FinePreprocess(_PackedCacheMixin, nn.Module):
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
        self._packed = None
        self._packed_key = None

    def _pack(self):
        ps = list(self.parameters())
        key = tuple(p._version for p in ps) + tuple(p.data_ptr() for p in ps)
        if self._packed is None or self._packed_key != key:
            with torch.no_grad():
                wm = self.merge_feat.weight.detach().float().contiguous()
                hi, lo, msc = split_weight(wm[:, : self.d_model_f])
                self._packed = {"wdt": self.down_proj.weight.detach().float().t().contiguous(),
                                "bd": self.down_proj.bias.detach().float().contiguous(),
                                "wm2t": wm[:, self.d_model_f:].t().contiguous(),
                                "bm": self.merge_feat.bias.detach().float().contiguous(),
                                "wm_hi": hi, "wm_lo": lo, "wm_scale": msc}
            self._packed_key = key
        return self._packed

    def run(self, feat_f0, feat_f1, feat_c_all, n, L, S, data, live=None):
        """-> _TokenState of the fine transformer (rows: side, match, window position), or None if M == 0.
        `live`: int32 device count; the match keys of `data` are then capacity buffers and only windows below the
        count are gathered (rows keep the capacity layout side*cap*WW + m*WW + k)."""
        lib = _lib.load()
        W = self.W
        stride = data["hw0_f"][0] // data["hw0_c"][0]
        data.update({"W": W})
        m = int(data["b_ids"].shape[0])
        if m == 0:
            return None
        p = self._pack()
        cf = self.d_model_f
        dev = feat_f0.device
        state = _TokenState(m * W * W, m * W * W, cf, dev)
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
        _lib.check(lib.lb_fine_preprocess(C.byref(a), ws.data_ptr(), nbytes, _stream(feat_f0)))
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
        if state is None:
            e = torch.empty(0, ww, self.d_model_f, device=feat_f0.device)
            return e, e.clone()
        m = state.rows0 // ww
        return state.x[: m * ww].view(m, ww, -1), state.x[m * ww:].view(m, ww, -1)


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

    def __init__(self, config, backbone_impl="auto"):
        """backbone_impl: "torch" keeps the PyTorch/cuDNN ResNet-FPN forward (the north_star default scope);
        "b200" runs it as implicit-GEMM convolutions on the tensor cores (SURVEY.md §8(f) rank 1); "auto" picks
        "b200" whenever the configured backbone is the supported ResNetFPN_8_2 shape.  Both are GPU paths."""
        super().__init__()
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
        if backbone_impl not in ("torch", "b200"):
            raise ValueError(backbone_impl)
        if backbone_impl == "b200" and not TensorCoreBackbone.supported(self.backbone):
            raise ValueError("the tensor-core backbone is built for ResNetFPN_8_2 with initial_dim 128, dims <= 256")
        self.backbone_impl = backbone_impl
        self._tc_backbone = TensorCoreBackbone(self.backbone) if backbone_impl == "b200" else None
        self.pos_encoding = PositionEncodingSine(config["coarse"]["d_model"],
                                                 temp_bug_fix=config["coarse"]["temp_bug_fix"])
        self.loftr_coarse = LocalFeatureTransformer(config["coarse"])
        self.coarse_matching = CoarseMatching(config["match_coarse"])
        self.fine_preprocess = FinePreprocess(config)
        self.loftr_fine = LocalFeatureTransformer(config["fine"])
        self.fine_matching = FineMatching()

    @torch.no_grad()
    def forward(self, data):
        """Updates `data` in place with the reference's keys; returns None.
        Inputs: image0/image1 [N, 1, H, W] float32 (H, W divisible by 8), optional mask0/mask1 [N, H/8, W/8],
        optional scale0/scale1 [N, 2]."""
        if self.training:
            raise NotImplementedError("loftr_b200 builds the inference path only: call .eval()")
        _require_cuda(data["image0"], "image0")
        state, feat_f0, feat_f1, bs, L, S, c, m0, m1 = self._coarse_features(data)
        img0 = data["image0"]

        # 3. coarse matching                                                           [loftr.py:67]
        self.coarse_matching.run(state.cat_hi, state.cat_lo, 2 * c, bs, L, S, c, data, m0, m1)

        # 4. fine-level refinement                                                     [loftr.py:70-72]
        fstate = self.fine_preprocess.run(feat_f0.float(), feat_f1.float(), state.x, bs, L, S, data)
        ww = self.fine_preprocess.W ** 2
        if fstate is not None:
            m = fstate.rows0 // ww
            self.loftr_fine.run(fstate, m, ww, ww)
            f0u, f1u = fstate.x[: m * ww].view(m, ww, -1), fstate.x[m * ww:].view(m, ww, -1)
        else:
            f0u = torch.empty(0, ww, self.fine_preprocess.d_model_f, device=img0.device)
            f1u = f0u.clone()

        # 5. fine matching                                                             [loftr.py:75]
        self.fine_matching(f0u, f1u, data)
        if self.expose_coarse_features:   # test / debugging tap, off by default: not a reference key
            data["_feat_c0"], data["_feat_c1"] = state.x[: bs * L].view(bs, L, c), state.x[bs * L:].view(bs, S, c)

    @torch.no_grad()
    def forward_static(self, data, capacity=None):
        """Sync-free, static-shape forward: the same inputs and keys as `forward`, without any host synchronisation,
        so that it can be captured by `torch.cuda.graph` (after one eager call, which packs the weights).

        Every input, masks and scales included, must already be on the device.  The match keys (b_ids, i_ids, j_ids,
        m_bids, gt_mask, mconf, mkpts0_c/1_c, mkpts0_f/1_f, expec_f) are fixed-capacity tensors with first dimension
        `capacity`, and data["num_matches"] is an int32 device tensor [1] with the true match count.  The count may
        exceed `capacity`; entries at or past min(count, capacity) are unspecified.  Only windows below the count are
        refined: the fine stage reads the count on the device.

        capacity: defaults to the exact bound of the coarse stage, n*min(L, S) (n*L with masks).  The fine stage keeps
        about 5 KB of state per window row, i.e. about 256 KB per match of capacity (about 10 GB at batch 8 640x480):
        a smaller capacity trades that memory for the risk of overflow, which stays visible in num_matches.

        Configurations whose output list depends on the data (match_coarse.thr < 0) raise ValueError."""
        if self.training:
            raise NotImplementedError("loftr_b200 builds the inference path only: call .eval()")
        if self.coarse_matching.thr < 0:
            raise ValueError("forward_static needs match_coarse.thr >= 0: with thr < 0 the reference's mconf != 0 "
                             "filter makes the output list depend on the data")
        if capacity is not None and int(capacity) < 1:
            raise ValueError(f"capacity must be a positive number of matches (got {capacity})")
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
        state, feat_f0, feat_f1, bs, L, S, c, m0, m1 = self._coarse_features(data)
        cap = self.coarse_matching.default_capacity(bs, L, S, m0 is not None) if capacity is None else int(capacity)

        # 3. coarse matching into capacity buffers; `count` stays on the device
        count = self.coarse_matching.run_static(state.cat_hi, state.cat_lo, 2 * c, bs, L, S, c, data, m0, m1, cap)

        # 4. fine-level refinement over the capacity layout, bounded on the device by `count`
        fstate = self.fine_preprocess.run(feat_f0.float(), feat_f1.float(), state.x, bs, L, S, data, live=count)
        ww = self.fine_preprocess.W ** 2
        self.loftr_fine.run(fstate, cap, ww, ww, live=count)
        f0u, f1u = fstate.x[: cap * ww].view(cap, ww, -1), fstate.x[cap * ww:].view(cap, ww, -1)

        # 5. fine matching
        self.fine_matching(f0u, f1u, data, live=count)
        if self.expose_coarse_features:
            data["_feat_c0"], data["_feat_c1"] = state.x[: bs * L].view(bs, L, c), state.x[bs * L:].view(bs, S, c)

    def _coarse_features(self, data):
        """Steps 1-2 of the forward (no host sync): backbone, position encoding and coarse transformer.
        -> (coarse token state, feat_f0, feat_f1, n, L, S, C, mask0 u8, mask1 u8)."""
        img0, img1 = data["image0"], data["image1"]
        lib = _lib.load()
        bs = img0.size(0)
        data.update({"bs": bs, "hw0_i": img0.shape[2:], "hw1_i": img1.shape[2:]})

        # 1. local feature CNN                                                         [loftr.py:45-49]
        nhwc = self._tc_backbone is not None
        if nhwc:   # NHWC outputs; viewed as [N, C, H, W] tensors with channels-last strides
            if data["hw0_i"] == data["hw1_i"]:
                fc, ff = self._tc_backbone(torch.cat([img0, img1], dim=0))
                (feat_c0, feat_c1), (feat_f0, feat_f1) = fc.split(bs), ff.split(bs)
            else:
                (feat_c0, feat_f0), (feat_c1, feat_f1) = self._tc_backbone(img0), self._tc_backbone(img1)
            feat_c0, feat_c1, feat_f0, feat_f1 = (t.permute(0, 3, 1, 2) for t in (feat_c0, feat_c1, feat_f0, feat_f1))
        elif data["hw0_i"] == data["hw1_i"]:
            feats_c, feats_f = self.backbone(torch.cat([img0, img1], dim=0))
            (feat_c0, feat_c1), (feat_f0, feat_f1) = feats_c.split(bs), feats_f.split(bs)
        else:
            (feat_c0, feat_f0), (feat_c1, feat_f1) = self.backbone(img0), self.backbone(img1)
        data.update({"hw0_c": feat_c0.shape[2:], "hw1_c": feat_c1.shape[2:],
                     "hw0_f": feat_f0.shape[2:], "hw1_f": feat_f1.shape[2:]})

        # 2. position encoding + token layout + coarse transformer                     [loftr.py:58-64]
        c = feat_c0.shape[1]
        (h0, w0), (h1, w1) = data["hw0_c"], data["hw1_c"]
        L, S = h0 * w0, h1 * w1
        state = _TokenState(bs * L, bs * S, c, img0.device)
        pe = self.pos_encoding.pe[0]
        st = _stream(img0)
        for feat, h, w, row0 in ((feat_c0, h0, w0, 0), (feat_c1, h1, w1, bs * L)):
            feat = feat.float()
            feat = feat.permute(0, 2, 3, 1).contiguous() if nhwc else feat.contiguous()   # no copy in either case
            _lib.check(lib.lb_coarse_prep(feat.data_ptr(), int(nhwc), pe.data_ptr(), bs, c, h, w, pe.shape[1], pe.shape[2],
                                          state.x.data_ptr() + row0 * c * 4,
                                          state.cat_hi.data_ptr() + row0 * 2 * c * 2,
                                          state.cat_lo.data_ptr() + row0 * 2 * c * 2, st))
        mask_all = m0 = m1 = None
        if "mask0" in data:
            m0 = data["mask0"].flatten(-2).reshape(-1).to(torch.uint8)
            m1 = data["mask1"].flatten(-2).reshape(-1).to(torch.uint8)
            mask_all = torch.cat([m0, m1]).contiguous()
            m0, m1 = mask_all[: bs * L], mask_all[bs * L:]
        self.loftr_coarse.run(state, bs, L, S, mask_all)
        return state, feat_f0, feat_f1, bs, L, S, c, m0, m1

    def invalidate_packed(self):
        """Drop every packed-weight cache (fp16 hi/lo planes, folded BatchNorm): required after parameter writes
        that PyTorch cannot see (`.data` mutation); implied by load_state_dict / .to() / .cuda() / .float()."""
        for m in self.modules():
            if m is not self and hasattr(m, "invalidate_packed"):
                m.invalidate_packed()
        if self._tc_backbone is not None:
            self._tc_backbone.invalidate_packed()

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


def _weight_refs(model):
    """(packed-weight cache objects, parameters + buffers, their (data_ptr, _version) key) of `model`: everything a
    captured graph holds raw device pointers into."""
    caches = [model.loftr_coarse._packed, model.loftr_fine._packed, model.fine_preprocess._packed]
    if model._tc_backbone is not None:
        caches.append(model._tc_backbone._packed)
    tensors = list(model.parameters()) + list(model.buffers())
    return caches, tensors, tuple((t.data_ptr(), t._version) for t in tensors)


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
    stale weights; `recapture()` rebuilds the graph.  See `LoFTR.forward_static` for `capacity` and its memory cost."""

    _TRIMMED = ("b_ids", "i_ids", "j_ids", "gt_mask", "mconf", "mkpts0_c", "mkpts1_c", "mkpts1_f", "expec_f")

    def __init__(self, model, batch, hw0, hw1=None, masks=False, scales=False, capacity=None):
        if model.training:
            raise NotImplementedError("loftr_b200 builds the inference path only: call .eval()")
        if model.coarse_matching.thr < 0:
            raise ValueError("CapturedMatcher needs match_coarse.thr >= 0: with thr < 0 the reference's mconf != 0 "
                             "filter makes the output list depend on the data")
        if capacity is not None and int(capacity) < 1:
            raise ValueError(f"capacity must be a positive number of matches (got {capacity})")
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

    def _check_weights(self):
        caches, tensors, key = _weight_refs(self.model)
        c0, t0, k0 = self._refs
        if len(caches) != len(c0) or any(a is not b for a, b in zip(caches, c0)) or len(tensors) != len(t0) or \
                any(a is not b for a, b in zip(tensors, t0)) or key != k0:
            raise RuntimeError("loftr_b200.CapturedMatcher: weights changed since capture (load_state_dict, .to(), "
                               "invalidate_packed() or a parameter update); call recapture()")

    def __call__(self, data):
        if self.graph is None:
            raise RuntimeError("loftr_b200.CapturedMatcher: no captured graph; call recapture()")
        self._check_weights()
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
