"""float64 numpy statement of the image front end (DESIGN.md §14), written from its definition and independent of
loftr_b200/preprocess.py: grey conversion, target size, bilinear resize, canvas, 1/8 mask and scale.  The GPU tests
compare the kernel with it; the CPU tests compare it with the goldens of the reference pipeline and OpenCV."""
import numpy as np


def grey(img, channel_order="rgb"):
    """uint8 [h, w] or [h, w, 1|3] -> integer grey levels [h, w] (OpenCV's 15-bit fixed-point luma for colour)."""
    img = np.asarray(img)
    if img.ndim == 2 or img.shape[2] == 1:
        return img.reshape(img.shape[0], img.shape[1]).astype(np.int64)
    c = img.astype(np.int64)
    r, b = (c[..., 0], c[..., 2]) if channel_order == "rgb" else (c[..., 2], c[..., 0])
    return (9798 * r + 19235 * c[..., 1] + 3735 * b + 16384) >> 15


def target_size(w, h, resize=None, df=8):
    if resize is None:
        w_new, h_new = w, h
    elif isinstance(resize, (tuple, list)):
        w_new, h_new = resize
    else:
        scale = resize / max(h, w)
        w_new, h_new = int(round(w * scale)), int(round(h * scale))
    if df is not None:
        w_new, h_new = int(w_new // df * df), int(h_new // df * df)
    if w_new <= 0 or h_new <= 0:
        raise ValueError((w, h, resize, df))
    return w_new, h_new


def _taps(n_src, n_dst):
    s = (np.arange(n_dst) + 0.5) * (n_src / n_dst) - 0.5
    i0 = np.floor(s)
    f = s - i0
    i0 = i0.astype(np.int64)
    return np.clip(i0, 0, n_src - 1), np.clip(i0 + 1, 0, n_src - 1), f


def resize_levels(g, w_new, h_new):
    """Grey levels [h, w] -> float64 [h_new, w_new]: bilinear, half-pixel centres, edge clamp, not rounded."""
    g = np.asarray(g, np.float64)
    y0, y1, fy = _taps(g.shape[0], h_new)
    x0, x1, fx = _taps(g.shape[1], w_new)
    top = g[y0][:, x0] + fx * (g[y0][:, x1] - g[y0][:, x0])
    bot = g[y1][:, x0] + fx * (g[y1][:, x1] - g[y1][:, x0])
    return top + fy[:, None] * (bot - top)


def prepare(images, resize=None, df=8, pad_to=None, channel_order="rgb"):
    """-> dict(image float64 [K, 1, H, W], mask bool [K, H/8, W/8] or None, scale float32 [K, 2], size int32 [K, 2])."""
    sizes = [target_size(im.shape[1], im.shape[0], resize, df) for im in images]
    if pad_to is None:
        assert len(set(sizes)) == 1, sizes
        H, W = sizes[0][1], sizes[0][0]
    elif pad_to == "square":
        assert len({max(s) for s in sizes}) == 1, sizes
        H = W = max(sizes[0])
    elif pad_to == "batch":
        H, W = max(s[1] for s in sizes), max(s[0] for s in sizes)
    else:
        H, W = pad_to
    K = len(images)
    image = np.zeros((K, 1, H, W), np.float64)
    full = np.zeros((K, H, W), bool)
    for k, (im, (w_new, h_new)) in enumerate(zip(images, sizes)):
        image[k, 0, :h_new, :w_new] = resize_levels(grey(im, channel_order), w_new, h_new) / 255.0
        full[k, :h_new, :w_new] = True
    mask = full[:, ::8, ::8] if pad_to is not None else None   # nearest at 1/8 samples pixel (8y, 8x)
    scale = np.asarray([[im.shape[1] / s[0], im.shape[0] / s[1]] for im, s in zip(images, sizes)], np.float32)
    return {"image": image, "mask": mask, "scale": scale, "size": np.asarray(sizes, np.int32)}
