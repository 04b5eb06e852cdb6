"""Float64 emulation of the fp16 backbone (`backbone_impl="b200_fp16"`, lb_backbone_forward_fp16; DESIGN.md §15).

Every convolution after the stem multiplies the stored fp16 activation by fp16(w * 2^e) (e = `weight_exponent` of the
layer's weights, the exponent of the split path) and accumulates exactly; the epilogue applies 2^-e, the folded
BatchNorm, the residual, the FPN x2 bilinear upsample-add (align_corners=True) and the activation, in that order, and
the result is stored as one fp16 plane (round to nearest even).  Residual and upsample addends are the stored fp16
values.  The stem's product stays split (within fp32 of exact here) and only its output is rounded.  feat_c and
feat_f are the epilogue values before rounding (the kernels write them in fp32).

With rounding=False nothing is rounded and the emulation is the float64 ResNetFPN_8_2 forward, which pins its fold,
residual, upsample and activation structure."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _fold(bn, cout):
    if bn is None:
        return None, None
    scale = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    shift = bn.bias.detach().double() - bn.running_mean.detach().double() * scale
    return scale, shift


def backbone_fp16_ref(m, images, rounding=True):
    """m: the PyTorch ResNetFPN (depth 3); images [N, 1, H, W] -> (feat_c, feat_f) float64 NCHW, on the device of
    `images` (m must live there too)."""
    from loftr_b200.loftr import weight_exponent
    r16 = (lambda t: t.half().double()) if rounding else (lambda t: t)
    x = images.detach().double()

    def conv(inp, c, bn, act, res=None, up=None):
        w = c.weight.detach().float()
        if rounding:
            e = weight_exponent(w)
            acc = F.conv2d(inp, (w * 2.0 ** e).half().double(), stride=c.stride, padding=c.padding) * 2.0 ** (-e)
        else:
            acc = F.conv2d(inp, w.double(), stride=c.stride, padding=c.padding)
        y = _affine(acc, bn)
        if res is not None:
            y = y + res
        if up is not None:
            y = y + F.interpolate(up, scale_factor=2.0, mode="bilinear", align_corners=True)
        if act == "relu":
            y = F.relu(y)
        elif act == "leaky":
            y = F.leaky_relu(y, 0.01)
        return y

    def unit(inp, u):
        t = r16(conv(inp, u.conv1, u.bn1, "relu"))
        skip = inp if u.downsample is None else r16(conv(inp, u.downsample[0], u.downsample[1], None))
        return r16(conv(t, u.conv2, u.bn2, "relu", res=skip))

    # the stem: split product, one stored plane
    s0 = r16(F.relu(_affine(F.conv2d(x, m.conv1.weight.detach().double(), stride=2, padding=3), m.bn1)))
    feats = []
    y = s0
    for layer in (m.layer1, m.layer2, m.layer3):
        for u in layer:
            y = unit(y, u)
        feats.append(y)
    x1, x2, x3 = feats
    feat_c = conv(x3, m.layer3_outconv, None, None)
    x2l = r16(conv(x2, m.layer2_outconv, None, None, up=r16(feat_c)))
    m2 = r16(conv(x2l, m.layer2_outconv2[0], m.layer2_outconv2[1], "leaky"))
    x2o = r16(conv(m2, m.layer2_outconv2[3], None, None))
    x1l = r16(conv(x1, m.layer1_outconv, None, None, up=x2o))
    m1 = r16(conv(x1l, m.layer1_outconv2[0], m.layer1_outconv2[1], "leaky"))
    feat_f = conv(m1, m.layer1_outconv2[3], None, None)
    return feat_c, feat_f


def _affine(y, bn):
    """y * scale + shift of the folded BatchNorm (identity without one)"""
    scale, shift = _fold(bn, y.shape[1])
    return y if scale is None else y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
