"""Image front end: uint8 camera frames of any size -> the matcher's input, on the GPU.

Replaces the per-image host work of the reference's dataset readers (src/utils/dataset.py: `read_megadepth_gray`
:94-125, `read_scannet_gray` :141-157, `get_resized_wh`, `get_divisible_wh`, `pad_bottom_right`) and the 1/8 mask of
src/datasets/megadepth.py:119-125 with one kernel launch per call (`lb_preprocess_images`, DESIGN.md §14):

    grey (OpenCV's BGR2GRAY / RGB2GRAY integers, at source resolution)
    -> bilinear resize to `target_size` (cv2.resize's INTER_LINEAR geometry, fp32, not rounded to a grey level)
    -> / 255 -> top-left in a zero canvas -> bool mask at 1/8 of the canvas, scale = [w / w_new, h / h_new].

There is no CPU implementation, like every other stage.  Nothing here synchronises with the host: sizes come from
tensor shapes, and what the kernel needs (a table of per-image descriptors) is uploaded from pinned memory.
"""
from __future__ import annotations

import ctypes as C
import numbers
from typing import NamedTuple, Optional

import torch

from . import _lib
from .loftr import _stream, check_rectify

class PreparedImages(NamedTuple):
    image: torch.Tensor            # [K, 1, H, W] float32 in [0, 1], zero outside each image's valid region
    mask: Optional[torch.Tensor]   # bool [K, H/8, W/8], or None when no padding was requested
    scale: torch.Tensor            # [K, 2] float32: [w / w_new, h / h_new], source pixels per resized pixel
    size: torch.Tensor             # [K, 2] int32: the valid (w_new, h_new) of each image inside the canvas


def _is_int(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, bool)


def target_size(w, h, resize=None, df=8):
    """(w_new, h_new) of a w x h image, as the reference's get_resized_wh + get_divisible_wh: `resize` None keeps the
    size, an int resizes the longer edge to it (Python `round`, ties to even), a (w, h) pair is taken literally; then
    both sides are truncated to a multiple of `df` (None: not truncated).  A result with a zero side raises."""
    if not (_is_int(w) and _is_int(h)) or w <= 0 or h <= 0:
        raise ValueError(f"target_size: the image size must be two positive ints (got w={w!r}, h={h!r})")
    if df is not None and (not _is_int(df) or df <= 0):
        raise ValueError(f"target_size: df must be a positive int or None (got {df!r})")
    if resize is None:
        w_new, h_new = w, h
    elif _is_int(resize):
        scale = resize / max(h, w)
        w_new, h_new = int(round(w * scale)), int(round(h * scale))
    elif isinstance(resize, (tuple, list)) and len(resize) == 2 and all(_is_int(v) for v in resize):
        w_new, h_new = resize
    else:
        raise ValueError(f"target_size: resize must be None, an int (longer edge) or a (w, h) pair (got {resize!r})")
    if df is not None:
        w_new, h_new = w_new // df * df, h_new // df * df
    if w_new <= 0 or h_new <= 0:
        raise ValueError(f"target_size: a {w}x{h} image with resize={resize!r}, df={df} would become {w_new}x{h_new}")
    return int(w_new), int(h_new)


def _as_list(images, name):
    """`images` as a list of [h, w] / [h, w, c] uint8 tensors, refusing what the kernel cannot read."""
    if torch.is_tensor(images):
        if images.dim() not in (3, 4):
            raise ValueError(f"{name}: one tensor must be [K, h, w] or [K, h, w, 3] (got {tuple(images.shape)}); pass "
                             "images of different sizes as a list")
        images = list(images.unbind(0))
    elif not isinstance(images, (list, tuple)):
        raise TypeError(f"{name}: expected a uint8 tensor or a list of uint8 tensors (got {type(images).__name__})")
    if len(images) == 0:
        raise ValueError(f"{name}: no images")
    for i, t in enumerate(images):
        if not torch.is_tensor(t):
            raise TypeError(f"{name}[{i}]: expected a tensor (got {type(t).__name__})")
        if t.dtype != torch.uint8:
            raise TypeError(f"{name}[{i}]: images must be uint8 (got {t.dtype}); float images already in [0, 1] go to "
                            "the matcher directly")
        if t.dim() not in (2, 3):
            raise ValueError(f"{name}[{i}]: an image must be [h, w] or [h, w, 3] (got {tuple(t.shape)})")
        if t.dim() == 3 and t.shape[2] not in (1, 3):
            raise ValueError(f"{name}[{i}]: {t.shape[2]} channels; only grey (1) and interleaved colour (3) are read")
        if t.shape[0] == 0 or t.shape[1] == 0:
            raise ValueError(f"{name}[{i}]: an image with a zero side ({tuple(t.shape)})")
        if t.stride(0) >= 2 ** 31 or t.shape[1] * 3 >= 2 ** 31:
            raise ValueError(f"{name}[{i}]: rows of 2 GiB or more are beyond the kernel's 32-bit row stride")
    return list(images)


def _r_index(channel_order):
    """Position of the red byte in a 3-channel pixel."""
    if channel_order not in ("rgb", "bgr"):
        raise ValueError(f"channel_order must be 'rgb' or 'bgr' (got {channel_order!r})")
    return 0 if channel_order == "rgb" else 2


def _canvas(imgs, resize, df, pad_to, name):
    """Host rule: per-image (w_new, h_new), the canvas (H, W) and whether a mask is written."""
    sizes = [target_size(t.shape[1], t.shape[0], resize, df) for t in imgs]
    if pad_to is None:
        if len(set(sizes)) != 1:
            raise ValueError(f"{name}: without pad_to every image must end up the same size, got (w, h) = "
                             f"{sorted(set(sizes))}; use pad_to='batch', 'square' or (H, W)")
        H, W = sizes[0][1], sizes[0][0]
    elif pad_to == "square":
        sides = sorted({max(s) for s in sizes})
        if len(sides) != 1:
            raise ValueError(f"{name}: pad_to='square' needs one square for the call, got sides {sides}; use "
                             "pad_to='batch' or (H, W)")
        H = W = sides[0]
    elif pad_to == "batch":
        H, W = max(s[1] for s in sizes), max(s[0] for s in sizes)
    elif isinstance(pad_to, (tuple, list)) and len(pad_to) == 2 and all(_is_int(v) for v in pad_to):
        H, W = int(pad_to[0]), int(pad_to[1])
        if H < max(s[1] for s in sizes) or W < max(s[0] for s in sizes):
            raise ValueError(f"{name}: pad_to=(H, W)={(H, W)} is smaller than an image: (w, h) = {sorted(set(sizes))}")
    else:
        raise ValueError(f"{name}: pad_to must be None, 'square', 'batch' or (H, W) (got {pad_to!r})")
    if H % 8 or W % 8:
        raise ValueError(f"{name}: the canvas {H}x{W} (H x W) must be divisible by 8, the coarse stride (df={df})")
    return sizes, H, W, pad_to is not None


def _device(imgs, device, name):
    """The CUDA device the call runs on: `device`, else the images' CUDA device, else the current one."""
    cuda = sorted({t.device for t in imgs if t.is_cuda}, key=str)
    if len(cuda) > 1:
        raise ValueError(f"{name}: images on different CUDA devices ({', '.join(map(str, cuda))})")
    dev = torch.device(device) if device is not None else (cuda[0] if cuda else torch.device("cuda"))
    if dev.type != "cuda":
        raise RuntimeError(f"{name}: the target device must be a CUDA (H100) device (got {dev}); the image front end has "
                           "no CPU implementation")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    if cuda and cuda[0] != dev:
        raise ValueError(f"{name}: images are on {cuda[0]}, the target device is {dev}")
    return dev


class _Plan:
    """What one call launches with: the device descriptor table and the constant outputs (scale, size)."""

    def __init__(self, imgs, sizes, H, W, masked, r_index, dev, cached):
        K = len(imgs)
        # host images travel through one pinned staging buffer and one asynchronous copy
        host = [i for i, t in enumerate(imgs) if not t.is_cuda]
        src = [None] * K   # (device address, row stride in bytes)
        if host:
            stage = torch.empty(sum(imgs[i].numel() for i in host), dtype=torch.uint8, pin_memory=True)
            off = 0
            offs = {}
            for i in host:
                n = imgs[i].numel()
                stage[off:off + n].view(imgs[i].shape).copy_(imgs[i])
                offs[i], off = off, off + n
            self.stage = stage.to(dev, non_blocking=True)   # alive until the launch is enqueued
            for i in host:
                ch = imgs[i].shape[2] if imgs[i].dim() == 3 else 1
                src[i] = (self.stage.data_ptr() + offs[i], imgs[i].shape[1] * ch)
        self.views = []
        for i, t in enumerate(imgs):
            if not t.is_cuda:
                continue
            ch = t.shape[2] if t.dim() == 3 else 1
            if t.stride(-1) != 1 or (t.dim() == 3 and t.stride(1) != ch):   # the kernel steps rows only
                if cached:
                    raise ValueError("prepare_images: with descs= every image must have densely packed pixels within a "
                                     "row (the table holds its address)")
                t = t.contiguous()
            self.views.append(t)
            src[i] = (t.data_ptr(), t.stride(0))
        table = (_lib.LbImageDesc * K)()
        for i, (t, (w_new, h_new)) in enumerate(zip(imgs, sizes)):
            d = table[i]
            d.src, d.row_stride_bytes = src[i]
            d.h, d.w = t.shape[0], t.shape[1]
            d.channels = t.shape[2] if t.dim() == 3 else 1
            d.r_index = r_index
            d.h_new, d.w_new = h_new, w_new
        nb = C.sizeof(table)   # 40 bytes per descriptor: the float / int views below stay aligned
        blob = torch.empty(nb + 16 * K, dtype=torch.uint8, pin_memory=True)
        blob[:nb].copy_(torch.frombuffer(table, dtype=torch.uint8))
        blob[nb:nb + 8 * K].view(torch.float32).copy_(torch.tensor(
            [[t.shape[1] / s[0], t.shape[0] / s[1]] for t, s in zip(imgs, sizes)], dtype=torch.float32).view(-1))
        blob[nb + 8 * K:].view(torch.int32).copy_(torch.tensor(sizes, dtype=torch.int32).view(-1))
        self.blob = blob.to(dev, non_blocking=True)
        self.scale = self.blob[nb:nb + 8 * K].view(torch.float32).view(K, 2)
        self.size = self.blob[nb + 8 * K:].view(torch.int32).view(K, 2)
        self.K, self.H, self.W, self.masked, self.dev = K, H, W, masked, dev
        self.resized = any((t.shape[1], t.shape[0]) != s for t, s in zip(imgs, sizes))

    def run(self):
        image = torch.empty((self.K, 1, self.H, self.W), dtype=torch.float32, device=self.dev)
        mask = torch.empty((self.K, self.H // 8, self.W // 8), dtype=torch.bool, device=self.dev) if self.masked else None
        _lib.check(_lib.load().lb_preprocess_images(self.blob.data_ptr(), self.K, image.data_ptr(), self.H, self.W,
                                                    _lib.ptr(mask), _stream(self.dev)))
        return PreparedImages(image, mask, self.scale, self.size)


def _prepare(imgs, sizes, H, W, masked, r_index, dev, descs):
    if descs is None:
        return _Plan(imgs, sizes, H, W, masked, r_index, dev, cached=False)
    if not isinstance(descs, dict):
        raise TypeError("prepare_images: descs must be a dict the caller keeps between calls")
    if any(not t.is_cuda for t in imgs):
        raise ValueError("prepare_images: descs= caches device addresses, so every image must already be on the device")
    key = (tuple((t.data_ptr(), tuple(t.shape), t.stride()) for t in imgs), tuple(sizes), H, W, masked, r_index, dev)
    if key not in descs:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("prepare_images: these images are not in descs yet; call once with the same tensors and "
                               "descs before capturing a CUDA graph (the table is uploaded from host memory)")
        descs[key] = _Plan(imgs, sizes, H, W, masked, r_index, dev, cached=True)
    return descs[key]


def prepare_images(images, resize=None, df=8, pad_to=None, channel_order="rgb", device=None, descs=None):
    """uint8 images -> PreparedImages (image, mask, scale, size) on the GPU, in one kernel launch.

    images: one uint8 tensor [K, h, w] / [K, h, w, 3], or a list of [h, w] / [h, w, 3] uint8 tensors of any sizes, each
        on the GPU or on the host (host images are uploaded as uint8 through one pinned buffer).  Rows may be strided
        (a cropped view, a row-padded decoder buffer); pixels within a row must be dense or the image is copied.
    resize, df: see `target_size`.  channel_order: 'rgb' or 'bgr' for 3-channel images.
    pad_to: None - every image must end up the same size, no mask; 'square' - a max(h_new, w_new) square (the
        reference's img_padding); 'batch' - the per-axis maximum over the call; (H, W) - explicit, divisible by 8.
        Images sit top-left, the padding is 0.0, and mask[k, y, x] = (8y < h_new and 8x < w_new).
    device: the CUDA device to run on (default: the images' device, else the current CUDA device).
    descs: a dict kept by the caller.  The descriptor table of a call is stored in it under the images' addresses,
        shapes and options and reused by the next identical call, which then copies nothing from the host and can be
        captured by `torch.cuda.graph` (device-resident images only; scale and size are then the same tensors on
        every call; a call on another stream than the first must be ordered after it, as for any tensor).
    The result equals `img.float() / 255` (a true division) bit for bit when no image changes size.  `scale` is what
    the matcher takes as scale0 / scale1 to report keypoints in source-image pixels."""
    _lib.require(_lib.PREPROCESS_VERSION, "prepare_images")
    imgs = _as_list(images, "prepare_images")
    r_index = _r_index(channel_order)
    canvas = _canvas(imgs, resize, df, pad_to, "prepare_images")
    return _prepare(imgs, *canvas, r_index, _device(imgs, device, "prepare_images"), descs).run()


def prepare_pairs(images0, images1, resize=None, df=8, pad_to=None, channel_order="rgb", device=None, descs=None):
    """Both sides of a batch of pairs through `prepare_images` (same options; each side has its own canvas) -> the dict
    `matcher(data)` / `forward_static` take: image0, image1; mask0, mask1 when padding was requested; scale0, scale1
    when any image of either side changed size, so that mkpts0_f / mkpts1_f come back in source-image pixels."""
    _lib.require(_lib.PREPROCESS_VERSION, "prepare_pairs")
    imgs0, imgs1 = _as_list(images0, "prepare_pairs: images0"), _as_list(images1, "prepare_pairs: images1")
    if len(imgs0) != len(imgs1):
        raise ValueError(f"prepare_pairs: {len(imgs0)} images0 but {len(imgs1)} images1")
    r_index = _r_index(channel_order)
    c0 = _canvas(imgs0, resize, df, pad_to, "prepare_pairs: images0")
    c1 = _canvas(imgs1, resize, df, pad_to, "prepare_pairs: images1")
    dev = _device(imgs0 + imgs1, device, "prepare_pairs")
    plan0 = _prepare(imgs0, *c0, r_index, dev, descs)
    plan1 = _prepare(imgs1, *c1, r_index, dev, descs)
    p0, p1 = plan0.run(), plan1.run()
    data = {"image0": p0.image, "image1": p1.image}
    if p0.mask is not None:
        data["mask0"], data["mask1"] = p0.mask, p1.mask
    if plan0.resized or plan1.resized:
        data["scale0"], data["scale1"] = p0.scale, p1.scale
    return data


def warp_images(images1, model, hw, scale0=None, scale1=None):
    """image1 of every pair resampled onto image0's canvas through the pair's homography (DESIGN.md §19): the input
    that `matcher(data)` substitutes for image1 when data["rectify1"] is given, in one kernel launch and without a host
    sync.

    images1: float32 [N, 1, H1, W1] CUDA.  model: float32 [N, 3, 3] on the same device, x1 ~ H x0 in the coordinates
    of mkpts0_f / mkpts1_f (source pixels when scales are given; a model with a non-finite entry stands for the
    identity).  hw: image0's canvas (H, W), both positive multiples of 8.  scale0 / scale1: optional [N, 2] scales of
    image0 / image1 (both or neither).
    -> float32 [N, 1, H, W]: output pixel (x, y) is image1 sampled bilinearly at H (x sx0, y sy0) / (sx1, sy1), taps
    outside image1 read as 0 (grid_sample with align_corners=True and zero padding), and 0 beyond the horizon."""
    if not torch.is_tensor(images1) or images1.dtype != torch.float32 or images1.dim() != 4 or images1.shape[1] != 1:
        got = (images1.dtype, tuple(images1.shape)) if torch.is_tensor(images1) else type(images1).__name__
        raise ValueError(f"warp_images: images1 must be a float32 tensor [N, 1, H1, W1] (got {got})")
    n = images1.shape[0]
    if not (isinstance(hw, (tuple, list, torch.Size)) and len(hw) == 2 and all(_is_int(v) and v > 0 and v % 8 == 0
                                                                                for v in hw)):
        raise ValueError(f"warp_images: hw must be (H, W), positive multiples of 8 (got {hw!r})")
    if (scale0 is None) != (scale1 is None):
        raise ValueError("warp_images: give scale0 and scale1 together")
    scales = []
    for name, s in (("scale0", scale0), ("scale1", scale1)):
        if s is not None:
            if not torch.is_tensor(s) or tuple(s.shape) != (n, 2):
                raise ValueError(f"warp_images: {name} must be a tensor [N, 2] with N = {n}")
            s = s.to(images1.device, torch.float32).contiguous()
        scales.append(s)
    model = check_rectify(model, n, images1.device, "warp_images")   # on images1's device, which is then a CUDA one
    H, W = int(hw[0]), int(hw[1])
    images1 = images1.contiguous()
    out = torch.empty(n, 1, H, W, dtype=torch.float32, device=images1.device)
    _lib.check(_lib.load().lb_rectify_images(images1.data_ptr(), n, images1.shape[2], images1.shape[3],
                                             model.data_ptr(), _lib.ptr(scales[0]), _lib.ptr(scales[1]),
                                             out.data_ptr(), H, W, _stream(images1)))
    return out


def rotation_candidates(size0, size1, scale0=None, scale1=None):
    """The four quarter turns of image1 relative to image0, as data["rectify1_candidates"] of a rectification search
    (DESIGN.md §20): for a camera rolled by an unknown multiple of 90 degrees.  Torch operations on size0's device, no
    host sync.

    size0 / size1: [N, 2] valid (w, h) of image0 / image1 in network pixels (`PreparedImages.size`, or the canvas).
    scale0 / scale1: optional [N, 2] scales of image0 / image1 (both or neither), as forward's.
    -> float32 [N, 4, 3, 3]: candidate q is H_q = S1 T(c1) R^q T(-c0) S0^-1, formed in float64, with c = ((w - 1) / 2,
    (h - 1) / 2) of each image, R = [[0, 1], [-1, 0]] and S = diag(sx, sy, 1) (the identity without scales).  Without
    scales, image1 = torch.rot90(image0, q, dims=(-2, -1)) warped through candidate q (`warp_images`) is image0 bit
    for bit, for square and non-square images alike."""
    sizes = []
    for name, s in (("size0", size0), ("size1", size1)):
        if not torch.is_tensor(s) or s.dim() != 2 or s.shape[1] != 2 or s.dtype == torch.bool or s.is_complex():
            raise ValueError(f"rotation_candidates: {name} must be a real tensor [N, 2] of (w, h) (got "
                             f"{tuple(s.shape) if torch.is_tensor(s) else type(s).__name__})")
        sizes.append(s)
    n, dev = size0.shape[0], size0.device
    if size1.shape[0] != n:
        raise ValueError(f"rotation_candidates: size0 and size1 must have the same N (got {n} and {size1.shape[0]})")
    if (scale0 is None) != (scale1 is None):
        raise ValueError("rotation_candidates: give scale0 and scale1 together")
    f64 = torch.float64
    if scale0 is None:
        scale0 = scale1 = torch.ones(n, 2, dtype=f64, device=dev)
    for name, s in (("scale0", scale0), ("scale1", scale1)):
        if not torch.is_tensor(s) or tuple(s.shape) != (n, 2):
            raise ValueError(f"rotation_candidates: {name} must be a tensor [N, 2] with N = {n}")
    one = torch.ones(n, 1, dtype=f64, device=dev)

    def shift(c):   # T(c) [N, 3, 3]
        t = torch.eye(3, dtype=f64, device=dev).repeat(n, 1, 1)
        t[:, :2, 2] = c
        return t

    c0, c1 = ((s.to(dev, f64) - 1) / 2 for s in sizes)
    s0_inv = torch.diag_embed(torch.cat([1 / scale0.to(dev, f64), one], 1))
    s1 = torch.diag_embed(torch.cat([scale1.to(dev, f64), one], 1))
    q = torch.arange(4, dtype=f64, device=dev)
    cos, sin = (1 - q % 2) * (1 - q), (q % 2) * (2 - q)   # (1, 0, -1, 0), (0, 1, 0, -1): R^q, exactly
    r = torch.zeros(4, 3, 3, dtype=f64, device=dev)
    r[:, 0, 0], r[:, 0, 1], r[:, 1, 0], r[:, 1, 1], r[:, 2, 2] = cos, sin, -sin, cos, 1
    h = (s1 @ shift(c1))[:, None] @ r[None] @ (shift(-c0) @ s0_inv)[:, None]
    return (h + 0.0).float().contiguous()   # + 0.0: no negative zeros
