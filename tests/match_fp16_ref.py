"""Float64 emulation of the single-pass fp16 matching mode (`match_precision="fp16"`, lb_transformer_forward_fp16 /
lb_coarse_match_fp16; DESIGN.md §16).

Every tensor-core product of the coarse transformer, the fine transformer and the coarse score matrix multiplies the
hi planes of its operands and accumulates exactly:
- an activation operand is fp16(x) (round to nearest even) of the value the split path stores as hi + lo;
- a weight operand is fp16(w * 2^e) * 2^-e, with e = `weight_exponent` of the packed matrix (q|k|v share the exponent
  of their concatenation, as in `LocalFeatureTransformer._build`);
- coarse linear attention: K^T V and Ksum from fp16(K) and fp16(V), K = elu(k)+1 and V masked; Q stays exact;
- coarse full attention: S = fp16(Q) fp16(K)^T, P = exp(S / sqrt(D) - rowmax) rounded once to fp16 in the product
  with fp16(V), the row sum taken from the unrounded P;
- the fine (window) attention stays exact: the window kernels run in fp32 on the fp32 projections;
- score matrix: fp16(feat_c0) . fp16(feat_c1), shared by every pass.
Epilogues, LayerNorm, residuals, masks and everything after the score matrix are those of `ref64`.

With `rounding=False` every rounding is the identity and each function equals its `ref64` counterpart."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import ref64

F64 = torch.float64


def r16(t, rounding=True):
    """fp16 round to nearest even (the hi plane), back in float64."""
    return t.half().double() if rounding else t


def w16(w, e, rounding=True):
    """hi weight plane fp16(w * 2^e) as a value: fp16(w * 2^e) * 2^-e."""
    return (w * 2.0 ** e).half().double() * 2.0 ** (-e) if rounding else w


def layer_exponents(w):
    """weight_exponent of each packed matrix of one layer (`w`: ref64.layer_weights dict)."""
    from loftr_b200.loftr import weight_exponent
    qkv = torch.cat([w["q_proj.weight"], w["k_proj.weight"], w["v_proj.weight"]], 0).float()
    return {"qkv": weight_exponent(qkv), "merge": weight_exponent(w["merge.weight"].float()),
            "mlp0": weight_exponent(w["mlp.0.weight"].float()), "mlp2": weight_exponent(w["mlp.2.weight"].float())}


def linear_attention(q, k, v, q_mask=None, kv_mask=None, eps=1e-6, rounding=True):
    """ref64.linear_attention with K and V rounded to fp16 for K^T V and Ksum (kv_gemm_fp16_kernel)."""
    Q = F.elu(q) + 1
    K = F.elu(k) + 1
    if q_mask is not None:
        Q = Q * q_mask[:, :, None, None].to(F64)
    if kv_mask is not None:
        K = K * kv_mask[:, :, None, None].to(F64)
        v = v * kv_mask[:, :, None, None].to(F64)
    K, v = r16(K, rounding), r16(v, rounding)
    KV = torch.einsum("nshd,nshv->nhdv", K, v)
    Z = 1 / (torch.einsum("nlhd,nhd->nlh", Q, K.sum(dim=1)) + eps)
    return torch.einsum("nlhd,nhdv,nlh->nlhv", Q, KV, Z)


def full_attention(q, k, v, q_mask=None, kv_mask=None, block=1024, rounding=True):
    """ref64.full_attention on fp16 Q, K, V with P rounded once to fp16 (full_attn_wgmma_fp16_kernel)."""
    q, k, v = r16(q, rounding), r16(k, rounding), r16(v, rounding)
    n, L, H, D = q.shape
    out = torch.zeros(n, L, H, D, dtype=F64, device=q.device)
    for lo in range(0, L, block):
        hi = min(lo + block, L)
        s = torch.einsum("nlhd,nshd->nlsh", q[:, lo:hi], k) / math.sqrt(D)
        if kv_mask is not None:
            ok = q_mask[:, lo:hi, None, None] & kv_mask[:, None, :, None]
            s = s.masked_fill(~ok, float("-inf"))
        m = s.amax(dim=2, keepdim=True)
        p = torch.exp(s - torch.where(torch.isinf(m), torch.zeros_like(m), m))
        den = p.sum(dim=2)[..., None]                                   # [n, l, h, 1]; 0: no valid key
        num = torch.einsum("nlsh,nshd->nlhd", r16(p, rounding), v)
        out[:, lo:hi] = torch.where(den > 0, num / den.clamp_min(1e-300), torch.zeros_like(num))
    return out


def encoder_layer(x, source, w, nhead, x_mask=None, source_mask=None, attention="linear", rounding=True):
    """ref64.encoder_layer with every projection, merge and MLP product on fp16 operands.  The attention is rounded
    as above for the coarse transformer (head dim 32) and exact for the fine (window) transformer."""
    bs, _, c = x.shape
    dim = c // nhead
    e = layer_exponents(w)
    xh, sh = r16(x, rounding), r16(source, rounding)
    q = (xh @ w16(w["q_proj.weight"], e["qkv"], rounding).T).view(bs, -1, nhead, dim)
    k = (sh @ w16(w["k_proj.weight"], e["qkv"], rounding).T).view(bs, -1, nhead, dim)
    v = (sh @ w16(w["v_proj.weight"], e["qkv"], rounding).T).view(bs, -1, nhead, dim)
    if dim == 32:
        att = linear_attention if attention == "linear" else full_attention
        msg = att(q, k, v, x_mask, source_mask, rounding=rounding)
    else:
        att = ref64.linear_attention if attention == "linear" else ref64.full_attention
        msg = att(q, k, v, x_mask, source_mask)
    msg = r16(msg.reshape(bs, -1, c), rounding) @ w16(w["merge.weight"], e["merge"], rounding).T
    msg = F.layer_norm(msg, (c,), w["norm1.weight"], w["norm1.bias"])
    h = torch.relu(r16(torch.cat([x, msg], 2), rounding) @ w16(w["mlp.0.weight"], e["mlp0"], rounding).T)
    msg = r16(h, rounding) @ w16(w["mlp.2.weight"], e["mlp2"], rounding).T
    msg = F.layer_norm(msg, (c,), w["norm2.weight"], w["norm2.bias"])
    return x + msg


def transformer(feat0, feat1, layers, layer_names, nhead, mask0=None, mask1=None, attention="linear", rounding=True):
    """ref64.transformer over the fp16 encoder layers."""
    for w, name in zip(layers, layer_names):
        if name == "self":
            feat0 = encoder_layer(feat0, feat0, w, nhead, mask0, mask0, attention, rounding)
            feat1 = encoder_layer(feat1, feat1, w, nhead, mask1, mask1, attention, rounding)
        elif name == "cross":
            feat0 = encoder_layer(feat0, feat1, w, nhead, mask0, mask1, attention, rounding)
            feat1 = encoder_layer(feat1, feat0, w, nhead, mask1, mask0, attention, rounding)
        else:
            raise KeyError(name)
    return feat0, feat1


def conf_matrix(feat_c0, feat_c1, mc, mask_c0=None, mask_c1=None, bin_score=None, rounding=True):
    """ref64.conf_matrix on the fp16 features: the scale 1/sqrt(C) (and 1/T) is applied to the exact product."""
    return ref64.conf_matrix(r16(feat_c0, rounding), r16(feat_c1, rounding), mc, mask_c0, mask_c1, bin_score)
