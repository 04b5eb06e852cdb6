"""The image front end on the GPU (`prepare_images` / `prepare_pairs`, kernel `preprocess_images_kernel`) against its
float64 statement (tests/preprocess_ref.py), at the kernel's own boundaries, and end to end in front of the matcher,
the feature bank and the captured static forward."""
import numpy as np
import pytest
import torch

import loftr_b200
import preprocess_ref as ref
import weights as W
from loftr_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 2e-6   # on the [0, 1] image: fp32 interpolation of levels 0..255 against float64
_INPUT_KEYS = ("image0", "image1", "mask0", "mask1", "scale0", "scale1")


def _noise(seed, h, w, c=1):
    rs = np.random.RandomState(seed)
    return rs.randint(0, 256, (h, w) if c == 1 else (h, w, c)).astype(np.uint8)


def _smooth(seed, h, w):
    """A uint8 image with structure at the scale of the coarse grid (random weights match it reproducibly)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 1, h // 12 + 3, w // 12 + 3, generator=g)
    img = torch.nn.functional.interpolate(low, size=(h, w), mode="bicubic", align_corners=False)
    return (img[0, 0].clamp(0, 1) * 255).round().to(torch.uint8)


def _check(p, imgs_np, label, **opts):
    """PreparedImages against the float64 reference: image within TOL, padding exactly 0, mask / scale / size exact."""
    want = ref.prepare(imgs_np, **opts)
    image = p.image.cpu().numpy().astype(np.float64)
    assert p.image.dtype == torch.float32 and image.shape == want["image"].shape, (label, image.shape)
    err = np.abs(image - want["image"]).max()
    assert err <= TOL, (label, err)
    for k, (w_new, h_new) in enumerate(want["size"]):
        assert not image[k, 0, h_new:].any() and not image[k, 0, :, w_new:].any(), (label, "padding")
    if want["mask"] is None:
        assert p.mask is None, label
    else:
        assert p.mask.dtype == torch.bool and np.array_equal(p.mask.cpu().numpy(), want["mask"]), (label, "mask")
    assert p.scale.dtype == torch.float32 and np.array_equal(p.scale.cpu().numpy(), want["scale"]), (label, "scale")
    assert p.size.dtype == torch.int32 and np.array_equal(p.size.cpu().numpy(), want["size"]), (label, "size")
    return err


def _model(name="indoor_ds", thr=0.0):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model = loftr_b200.LoFTR(loftr_b200.get_cfg(name, thr=thr), backbone_impl="b200").eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict({k: torch.from_numpy(v) for k, v in W.make_state(shapes, seed=0).items()})
    return model.to(DEV)


def _assert_bitwise(got, want, label, keys=None):
    keys = [k for k in want if k not in _INPUT_KEYS] if keys is None else keys
    assert [k for k in got if k not in _INPUT_KEYS] == [k for k in want if k not in _INPUT_KEYS], label
    for k in keys:
        if torch.is_tensor(want[k]):
            assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), f"{label}: {k} differs"
        else:
            assert got[k] == want[k], (label, k)


# name -> ((h, w, channels), resize, pad_to, channel_order)
KERNEL_CASES = {
    "down2x_scannet": ((968, 1296, 1), (640, 480), None, "rgb"),
    "down_nonint_rgb": ((1001, 777, 3), 832, "square", "rgb"),
    "up_square": ((300, 400, 1), 832, "square", "rgb"),
    "odd_bgr": ((101, 77, 3), 96, "batch", "bgr"),
    "tiny_up": ((9, 9, 1), 64, None, "rgb"),
    "down3x_rgb_explicit": ((480, 642, 3), 208, (160, 256), "rgb"),
}


@pytest.mark.parametrize("name", sorted(KERNEL_CASES))
def test_kernel_equals_the_float64_reference(name):
    (h, w, c), resize, pad_to, order = KERNEL_CASES[name]
    img = _noise(3, h, w, c)
    for place in ("cuda", "host"):
        t = torch.from_numpy(img).to(DEV) if place == "cuda" else torch.from_numpy(img)
        p = loftr_b200.prepare_images([t], resize=resize, pad_to=pad_to, channel_order=order, device=DEV)
        _check(p, [img], f"{name}/{place}", resize=resize, pad_to=pad_to, channel_order=order)


@pytest.mark.parametrize("c", [1, 3])
def test_sliced_view_with_a_row_stride_and_a_width_off_the_float4_grid(c):
    base = _noise(5, 70, 131, c)
    t = torch.from_numpy(base).to(DEV)[3:67, 5:122]          # 64 x 117, row stride 131 * c
    assert not t.is_contiguous() and t.shape[1] % 4 != 0
    for resize in (None, 104, 200):
        p = loftr_b200.prepare_images([t], resize=resize, pad_to="batch", channel_order="bgr")
        _check(p, [base[3:67, 5:122]], f"view c={c} resize={resize}", resize=resize, pad_to="batch", channel_order="bgr")
    cols = torch.from_numpy(base).to(DEV)[:, ::2]             # a pixel stride the kernel does not step: copied
    _check(loftr_b200.prepare_images([cols]), [base[:, ::2]], f"strided pixels c={c}")


def test_identity_size_is_level_over_255_bit_for_bit():
    img = torch.from_numpy(np.stack([_noise(s, 64, 80) for s in range(3)]))
    img[0].view(-1)[:256] = torch.arange(256, dtype=torch.uint8)   # every level
    want = img.float() / 255   # on the host: a true division, as the reference's readers do
    _lib.timing_enable(True)
    try:
        p = loftr_b200.prepare_images(img.to(DEV))
        torch.cuda.synchronize()
        tags = _lib.timing_collect()
    finally:
        _lib.timing_enable(False)
    assert tags["preprocess"][1] == 1 and tags["preprocess"][0] > 0
    assert p.image.shape == (3, 1, 64, 80) and torch.equal(p.image.cpu()[:, 0], want)
    assert p.mask is None and torch.equal(p.scale.cpu(), torch.ones(3, 2))
    colour = torch.from_numpy(np.stack([_noise(9, 64, 80, 3)]))
    pc = loftr_b200.prepare_images(colour, channel_order="bgr", device=DEV)
    grey = torch.from_numpy(ref.grey(colour[0].numpy(), "bgr")).float() / 255
    assert torch.equal(pc.image.cpu()[0, 0], grey)
    # a padded canvas keeps the valid region exact and writes a mask
    pp = loftr_b200.prepare_images(img.to(DEV), pad_to=(72, 128))
    assert torch.equal(pp.image.cpu()[:, 0, :64, :80], want) and not pp.image[:, 0, 64:].any()
    assert not pp.image[:, 0, :, 80:].any() and pp.mask.shape == (3, 9, 16)
    assert pp.mask[:, :8, :10].all() and not pp.mask[:, 8:].any() and not pp.mask[:, :, 10:].any()


@pytest.mark.parametrize("mode", ["square", "batch", "explicit", "single"])
def test_ragged_list_equals_the_per_image_results(mode):
    specs = [(120, 160, 1, "cuda"), (200, 150, 3, "host"), (90, 90, 1, "host"), (64, 200, 3, "cuda")]
    if mode == "single":
        specs = specs[1:2]
    np_imgs = [_noise(20 + i, h, w, c) for i, (h, w, c, _) in enumerate(specs)]
    imgs = [torch.from_numpy(a).to(DEV) if s[3] == "cuda" else torch.from_numpy(a) for a, s in zip(np_imgs, specs)]
    resize, pad_to = {"square": (96, "square"), "batch": (None, "batch"), "explicit": (100, (104, 136)),
                      "single": (96, "batch")}[mode]
    p = loftr_b200.prepare_images(imgs, resize=resize, pad_to=pad_to, device=DEV)
    _check(p, np_imgs, mode, resize=resize, pad_to=pad_to)
    canvas = tuple(p.image.shape[2:])
    for k, t in enumerate(imgs):
        for one in (t, t.cpu(), t.to(DEV)):
            q = loftr_b200.prepare_images([one], resize=resize, pad_to=canvas, device=DEV)
            assert torch.equal(q.image[0], p.image[k]) and torch.equal(q.mask[0], p.mask[k]), (mode, k)
            assert torch.equal(q.scale[0], p.scale[k]) and torch.equal(q.size[0], p.size[k])


# ((h, w), df, pad_to (H, W)): canvas 8 wide; canvases off the 128-pixel tile; w_new ending inside a float4 and inside
# a mask cell's 8-pixel span (only reachable with df < 4: the canvas stays divisible by 8)
BOUNDARY_CASES = [((8, 8), 8, None), ((16, 8), 8, (24, 8)), ((40, 136), 8, None), ((24, 200), 8, (24, 264)),
                  ((37, 53), 1, (40, 56)), ((33, 49), 1, (40, 56)), ((31, 47), 1, (32, 48)), ((9, 130), 2, (16, 136)),
                  ((8, 127), 1, (8, 128)), ((8, 129), 1, (16, 256))]


@pytest.mark.parametrize("i", range(len(BOUNDARY_CASES)))
def test_canvas_widths_at_the_kernel_boundaries(i):
    (h, w), df, pad_to = BOUNDARY_CASES[i]
    for c in (1, 3):
        img = _noise(40 + i, h, w, c)
        p = loftr_b200.prepare_images([torch.from_numpy(img).to(DEV)], df=df, pad_to=pad_to)
        _check(p, [img], f"boundary {i} c={c}", df=df, pad_to=pad_to)
    # resized into the same canvas: the last valid column interpolates against the clamped edge
    if pad_to is not None and df == 1:
        img = _noise(60 + i, 3 * h + 1, 2 * w + 1)
        p = loftr_b200.prepare_images([torch.from_numpy(img)], resize=(w, h), df=1, pad_to=pad_to, device=DEV)
        _check(p, [img], f"boundary {i} resized", resize=(w, h), df=1, pad_to=pad_to)


def _torch_masks_and_scales(srcs, resize, canvas):
    """What a caller would build by hand (reference conventions): bool [n, H/8, W/8] masks, [w / w_new, h / h_new]."""
    H, W = canvas
    masks, scales = [], []
    for t in srcs:
        w_new, h_new = ref.target_size(t.shape[1], t.shape[0], resize, 8)
        full = torch.zeros(1, 1, H, W)
        full[..., :h_new, :w_new] = 1
        masks.append(torch.nn.functional.interpolate(full, scale_factor=0.125, mode="nearest",
                                                     recompute_scale_factor=False)[0, 0].bool())
        scales.append(torch.tensor([t.shape[1] / w_new, t.shape[0] / h_new], dtype=torch.float))
    return torch.stack(masks).to(DEV), torch.stack(scales).to(DEV)


def test_matcher_on_prepared_pairs_equals_a_hand_assembled_batch():
    """The sizes of the ds_masked_scaled case: 128 x 128 canvases, valid regions (128, 96), (104, 128) | (112, 128),
    (128, 88), reached from sources twice as large (one of them colour, one on the host)."""
    model = _model()
    src0 = [_smooth(1, 256, 192).to(DEV), _smooth(2, 208, 256)]
    src1 = [_smooth(3, 224, 256).to(DEV), _smooth(4, 256, 176).to(DEV)[..., None].expand(-1, -1, 3).contiguous()]
    data = loftr_b200.prepare_pairs(src0, src1, resize=128, pad_to="square", device=DEV)
    assert list(data) == ["image0", "image1", "mask0", "mask1", "scale0", "scale1"]
    assert data["image0"].shape == data["image1"].shape == (2, 1, 128, 128)
    hand = {"image0": data["image0"], "image1": data["image1"]}
    hand["mask0"], hand["scale0"] = _torch_masks_and_scales(src0, 128, (128, 128))
    hand["mask1"], hand["scale1"] = _torch_masks_and_scales(src1, 128, (128, 128))
    for k in ("mask0", "mask1", "scale0", "scale1"):
        assert data[k].dtype == hand[k].dtype and torch.equal(data[k], hand[k]), k
    model(data)
    model(hand)
    _assert_bitwise(data, hand, "prepared pairs")
    m = data["b_ids"].shape[0]
    assert m > 20
    # keypoints come back in source pixels; no match sits on a padded coarse cell
    for side, srcs, ids in ((0, src0, data["i_ids"]), (1, src1, data["j_ids"])):
        wh = torch.tensor([[t.shape[1], t.shape[0]] for t in srcs], dtype=torch.float, device=DEV)[data["b_ids"]]
        for key in (f"mkpts{side}_c", f"mkpts{side}_f"):
            pts = data[key]
            assert bool((pts >= 0).all()) and bool((pts < wh).all()), key
        assert bool(data[f"mask{side}"][data["b_ids"], ids // 16, ids % 16].all())
    # unresized pairs of one size: no masks, no scales, and the matcher's output for img.float() / 255
    same = [_smooth(7, 96, 128), _smooth(8, 96, 128)]
    d = loftr_b200.prepare_pairs(torch.stack(same).to(DEV), torch.stack(same[::-1]).to(DEV))
    assert list(d) == ["image0", "image1"]
    plain = {"image0": (torch.stack(same).float() / 255)[:, None].to(DEV),
             "image1": (torch.stack(same[::-1]).float() / 255)[:, None].to(DEV)}
    model(d)
    model(plain)
    _assert_bitwise(d, plain, "unresized pairs")


def test_feature_bank_of_mixed_photos_equals_prepared_pairs():
    model = _model()
    photos = [_smooth(11, 300, 400).to(DEV), _smooth(12, 420, 280), _smooth(13, 240, 240).to(DEV)]
    p = loftr_b200.prepare_images(photos, resize=160, pad_to="batch", device=DEV)
    assert p.image.shape == (3, 1, 160, 160) and p.mask.shape == (3, 20, 20)
    bank = model.extract_features(p.image, p.mask)
    i = torch.tensor([0, 1, 2, 2, 0], device=DEV)
    j = torch.tensor([1, 2, 0, 2, 0], device=DEV)
    got = model.match_features(bank, i, bank, j, scale0=p.scale, scale1=p.scale)
    data = loftr_b200.prepare_pairs([photos[k] for k in i.tolist()], [photos[k] for k in j.tolist()], resize=160,
                                    pad_to=(160, 160), device=DEV)
    model(data)
    _assert_bitwise(got, data, "bank of mixed photos")
    assert got["b_ids"].shape[0] > 20


def test_no_host_synchronisation_and_capture_with_forward_static():
    model = _model()
    n, h, w = 2, 200, 264

    def frames(seed):
        return (torch.stack([_smooth(seed + k, h, w) for k in range(n)]).to(DEV),
                torch.stack([_smooth(seed + 10 + k, h, w) for k in range(n)]).to(DEV))

    buf0, buf1 = frames(100)
    opts = dict(resize=128, pad_to="square")
    descs = {}

    def step():
        data = loftr_b200.prepare_pairs(buf0, buf1, descs=descs, **opts)
        model.forward_static(data)
        return data

    model(loftr_b200.prepare_pairs(buf0, buf1, **opts))   # packs the weights (that synchronises once)
    first = step()
    assert len(descs) == 2
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = step()
        uncached = loftr_b200.prepare_pairs(buf0, buf1, **opts)
        one = loftr_b200.prepare_images([buf0[0], buf1[1, 8:, :-3]], resize=96, pad_to="batch")
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(descs) == 2 and one.image.shape == (2, 1, 72, 96)
    for k in _INPUT_KEYS:
        assert torch.equal(again[k], first[k]) and torch.equal(uncached[k], first[k]), k
    assert again["scale0"] is first["scale0"]

    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="not in descs yet"):
        with torch.cuda.graph(g):
            loftr_b200.prepare_pairs(buf0, buf1, descs={}, **opts)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step()
    new0, new1 = frames(200)
    buf0.copy_(new0)
    buf1.copy_(new1)
    g.replay()
    torch.cuda.synchronize()
    eager = loftr_b200.prepare_pairs(new0, new1, **opts)
    model.forward_static(eager)
    m = int(eager["num_matches"].item())
    assert m > 20 and int(out["num_matches"].item()) == m
    assert not torch.equal(out["image0"], first["image0"])
    for k, v in eager.items():
        if not torch.is_tensor(v):
            assert out[k] == v, k
        elif v.dim() and v.shape[0] == eager["b_ids"].shape[0] and k not in _INPUT_KEYS:
            assert torch.equal(out[k][:m], v[:m]), k
        else:
            assert torch.equal(out[k], v), k
