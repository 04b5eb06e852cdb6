"""Float64 references of every hot-path stage -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Plain torch in float64, on whatever device the inputs live on, so that the GPU tests can judge the kernels at full size
next to them.  Each function restates one stage of the reference (zju3dv/LoFTR; file:line citations are relative to
the reference root).  Pinned against the reference's own float64 outputs by tests/test_ref64_cpu.py.

Conventions that differ from the reference:
- full attention gives a padded query row, and a row without any valid key, a zero message (the reference gives NaN;
  DESIGN.md §5).  Linear attention yields zero for both by construction.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

F64 = torch.float64
INF = 1e9  # coarse_matching.py:6


def f64(x, device=None):
    """array / tensor -> float64 tensor (on `device`, or where it already is)."""
    t = torch.as_tensor(x)
    return t.to(device=device if device is not None else t.device, dtype=F64)


# ------------------------------------------------------------------------------------------------ transformer
def linear_attention(q, k, v, q_mask=None, kv_mask=None, eps=1e-6):
    """LinearAttention.forward (linear_attention.py:20-47).  q [N,L,H,D], k / v [N,S,H,D]."""
    Q = F.elu(q) + 1                                                    # :31-32
    K = F.elu(k) + 1
    if q_mask is not None:                                              # :35-39
        Q = Q * q_mask[:, :, None, None].to(F64)
    if kv_mask is not None:
        K = K * kv_mask[:, :, None, None].to(F64)
        v = v * kv_mask[:, :, None, None].to(F64)
    v_length = v.shape[1]
    v = v / v_length                                                    # :41-42
    KV = torch.einsum("nshd,nshv->nhdv", K, v)                          # :43
    Z = 1 / (torch.einsum("nlhd,nhd->nlh", Q, K.sum(dim=1)) + eps)     # :44
    return torch.einsum("nlhd,nhdv,nlh->nlhv", Q, KV, Z) * v_length    # :45


def full_attention(q, k, v, q_mask=None, kv_mask=None, block=1024):
    """FullAttention.forward (linear_attention.py:56-81), query-blocked, with the zero-message convention."""
    n, L, H, D = q.shape
    out = torch.zeros(n, L, H, D, dtype=F64, device=q.device)
    for lo in range(0, L, block):
        hi = min(lo + block, L)
        qk = torch.einsum("nlhd,nshd->nlsh", q[:, lo:hi], k)           # :69
        if kv_mask is not None:                                         # :70-71
            ok = q_mask[:, lo:hi, None, None] & kv_mask[:, None, :, None]
            qk = qk.masked_fill(~ok, float("-inf"))
        a = torch.softmax(qk / math.sqrt(D), dim=2)                     # :74-75
        a = torch.nan_to_num(a, nan=0.0)                                # rows without a valid logit: zero message
        out[:, lo:hi] = torch.einsum("nlsh,nshd->nlhd", a, v)           # :79
    return out


def encoder_layer(x, source, w, nhead, x_mask=None, source_mask=None, attention="linear"):
    """LoFTREncoderLayer.forward (transformer.py:35-58).  `w`: the layer's state_dict suffixes -> float64 tensors."""
    bs, _, c = x.shape
    dim = c // nhead
    q = (x @ w["q_proj.weight"].T).view(bs, -1, nhead, dim)             # :47
    k = (source @ w["k_proj.weight"].T).view(bs, -1, nhead, dim)        # :48
    v = (source @ w["v_proj.weight"].T).view(bs, -1, nhead, dim)        # :49
    att = linear_attention if attention == "linear" else full_attention
    msg = att(q, k, v, x_mask, source_mask)                             # :50
    msg = msg.reshape(bs, -1, c) @ w["merge.weight"].T                  # :51
    msg = F.layer_norm(msg, (c,), w["norm1.weight"], w["norm1.bias"])   # :52
    msg = torch.relu(torch.cat([x, msg], 2) @ w["mlp.0.weight"].T) @ w["mlp.2.weight"].T   # :55
    msg = F.layer_norm(msg, (c,), w["norm2.weight"], w["norm2.bias"])   # :56
    return x + msg                                                      # :58


def layer_weights(tf_module, device=None):
    """float64 per-layer weight dicts of a loftr_b200 LocalFeatureTransformer (same names as the reference)."""
    sd = tf_module.state_dict()
    out = []
    for i in range(len(tf_module.layers)):
        pre = f"layers.{i}."
        out.append({k[len(pre):]: f64(v, device) for k, v in sd.items() if k.startswith(pre)})
    return out


def transformer(feat0, feat1, layers, layer_names, nhead, mask0=None, mask1=None, attention="linear"):
    """LocalFeatureTransformer.forward (transformer.py:80-101): feat1 attends to the updated feat0 (:96-97)."""
    for w, name in zip(layers, layer_names):
        if name == "self":
            feat0 = encoder_layer(feat0, feat0, w, nhead, mask0, mask0, attention)
            feat1 = encoder_layer(feat1, feat1, w, nhead, mask1, mask1, attention)
        elif name == "cross":
            feat0 = encoder_layer(feat0, feat1, w, nhead, mask0, mask1, attention)
            feat1 = encoder_layer(feat1, feat0, w, nhead, mask1, mask0, attention)
        else:
            raise KeyError(name)
    return feat0, feat1


# ------------------------------------------------------------------------------------------------ coarse matching
def log_optimal_transport(scores, alpha, iters):
    """log_optimal_transport + log_sinkhorn_iterations (superglue.py:141-170), any iters >= 0 -> [N, L+1, S+1]."""
    b, m, n = scores.shape
    alpha = f64(alpha, scores.device).reshape(())
    couplings = torch.cat([torch.cat([scores, alpha.expand(b, m, 1)], -1),
                           torch.cat([alpha.expand(b, 1, n), alpha.expand(b, 1, 1)], -1)], 1)   # :157-160
    norm = -math.log(m + n)                                                                    # :162
    log_mu = torch.tensor([norm] * m + [math.log(n) + norm], dtype=F64, device=scores.device)  # :163
    log_nu = torch.tensor([norm] * n + [math.log(m) + norm], dtype=F64, device=scores.device)  # :164
    u = torch.zeros(b, m + 1, dtype=F64, device=scores.device)
    v = torch.zeros(b, n + 1, dtype=F64, device=scores.device)
    for _ in range(iters):                                                                     # :144-147
        u = log_mu - torch.logsumexp(couplings + v[:, None, :], dim=2)
        v = log_nu - torch.logsumexp(couplings + u[:, :, None], dim=1)
    return couplings + u[:, :, None] + v[:, None, :] - norm                                    # :148,169


def conf_matrix(feat_c0, feat_c1, mc, mask_c0=None, mask_c1=None, bin_score=None):
    """CoarseMatching.forward up to conf_matrix (coarse_matching.py:103-143).  feat [N, L|S, C]; masks bool [N, L|S]."""
    c = feat_c0.shape[-1]
    f0, f1 = feat_c0 / c ** 0.5, feat_c1 / c ** 0.5                                         # :106-107
    pad = None if mask_c0 is None else ~(mask_c0[..., None] & mask_c1[:, None])
    if mc["match_type"] == "dual_softmax":
        sim = torch.einsum("nlc,nsc->nls", f0, f1) / mc["dsmax_temperature"]                 # :110
        if pad is not None:
            sim = sim.masked_fill(pad, -INF)                                                  # :111-114
        return torch.softmax(sim, 1) * torch.softmax(sim, 2)                                  # :115
    if mc["match_type"] == "sinkhorn":
        sim = torch.einsum("nlc,nsc->nls", f0, f1)                                            # :119
        if pad is not None:
            sim = sim.masked_fill(pad, -INF)                                                  # :120-123
        assign = log_optimal_transport(sim, bin_score, mc["skh_iters"]).exp()                # :126-128
        L, S = sim.shape[1:]
        conf = assign[:, :-1, :-1].clone()                                                    # :129
        if mc.get("skh_prefilter", False):                                                    # :132-136
            filter0 = (assign.argmax(dim=2) == S)[:, :-1]
            filter1 = (assign.argmax(dim=1) == L)[:, :-1]
            conf[filter0[..., None].expand_as(conf)] = 0
            conf[filter1[:, None].expand_as(conf)] = 0
        return conf
    raise NotImplementedError(mc["match_type"])


def coarse_match(conf, mc, hw0_i, hw0_c, hw1_c, mask0=None, mask1=None, scale0=None, scale1=None):
    """CoarseMatching.get_coarse_match, eval path (coarse_matching.py:8-43,150-197,238-261).
    mask0 / mask1: bool [N, h, w] grids (their presence selects the padded-extent border removal)."""
    n = conf.shape[0]
    (h0, w0), (h1, w1) = hw0_c, hw1_c
    m = (conf > mc["thr"]).reshape(n, h0, w0, h1, w1)                                       # :167
    bd = mc["border_rm"]
    if bd > 0:
        m[:, :bd] = False                                                                     # :18-21, :32-35
        m[:, :, :bd] = False
        m[:, :, :, :bd] = False
        m[:, :, :, :, :bd] = False
        if mask0 is None:                                                                     # :22-25
            m[:, -bd:] = False
            m[:, :, -bd:] = False
            m[:, :, :, -bd:] = False
            m[:, :, :, :, -bd:] = False
        else:                                                                                 # :37-43
            h0s, w0s = mask0.sum(1).max(-1)[0].int(), mask0.sum(-1).max(-1)[0].int()
            h1s, w1s = mask1.sum(1).max(-1)[0].int(), mask1.sum(-1).max(-1)[0].int()
            for b, (a0, b0, a1, b1) in enumerate(zip(h0s.tolist(), w0s.tolist(), h1s.tolist(), w1s.tolist())):
                m[b, a0 - bd:] = False
                m[b, :, b0 - bd:] = False
                m[b, :, :, a1 - bd:] = False
                m[b, :, :, :, b1 - bd:] = False
    m = m.reshape(conf.shape)
    m = m & (conf == conf.max(dim=2, keepdim=True)[0]) & (conf == conf.max(dim=1, keepdim=True)[0])   # :179-181
    mask_v, all_j = m.max(dim=2)                                                              # :185
    b_ids, i_ids = torch.where(mask_v)                                                        # :186
    j_ids = all_j[b_ids, i_ids]
    mconf = conf[b_ids, i_ids, j_ids]
    scale = hw0_i[0] / hw0_c[0]                                                               # :241
    s0 = scale * f64(scale0, conf.device)[b_ids] if scale0 is not None else scale
    s1 = scale * f64(scale1, conf.device)[b_ids] if scale1 is not None else scale
    mk0 = torch.stack([i_ids % w0, torch.div(i_ids, w0, rounding_mode="floor")], 1).to(F64) * s0   # :244-246
    mk1 = torch.stack([j_ids % w1, torch.div(j_ids, w1, rounding_mode="floor")], 1).to(F64) * s1   # :247-249
    return {"b_ids": b_ids, "i_ids": i_ids, "j_ids": j_ids, "mconf": mconf, "mkpts0_c": mk0, "mkpts1_c": mk1}


def top2(conf):
    """Adjudication statistics: the two largest confidences of every row and every column -> [N, L, 2], [N, S, 2].
    A dimension of size 1 contributes a zero second value."""
    def t2(x, dim):
        if x.shape[dim] >= 2:
            return torch.topk(x, 2, dim=dim).values
        return torch.cat([x, torch.zeros_like(x)], dim)
    return t2(conf, 2), t2(conf, 1).transpose(1, 2)


# ------------------------------------------------------------------------------------------------ fine level
def fine_windows(feat_f, b_ids, idx, W, stride):
    """F.unfold(kernel W, stride, padding W//2) + rearrange + [b_ids, idx] (fine_preprocess.py:40-47) -> [M, WW, C]."""
    u = F.unfold(feat_f, kernel_size=(W, W), stride=stride, padding=W // 2)                   # :40
    n, cww, l = u.shape
    u = u.view(n, cww // (W * W), W * W, l).permute(0, 3, 2, 1)                               # 'n (c ww) l -> n l ww c'
    return u[b_ids, idx]                                                                      # :46-47


def fine_preprocess(feat_f0, feat_f1, feat_c0, feat_c1, b_ids, i_ids, j_ids, W, stride, w):
    """FinePreprocess.forward, fine_concat_coarse_feat=True (fine_preprocess.py:29-59).  feat_f [N, C, H, W] float64;
    w: 'down_proj.weight/bias', 'merge_feat.weight/bias' float64."""
    win0 = fine_windows(feat_f0, b_ids, i_ids, W, stride)
    win1 = fine_windows(feat_f1, b_ids, j_ids, W, stride)
    c_win = torch.cat([feat_c0[b_ids, i_ids], feat_c1[b_ids, j_ids]], 0) @ w["down_proj.weight"].T + w["down_proj.bias"]
    cat = torch.cat([torch.cat([win0, win1], 0), c_win[:, None].expand(-1, W * W, -1)], -1)  # :52-55
    merged = cat @ w["merge_feat.weight"].T + w["merge_feat.bias"]
    m = len(b_ids)
    return merged[:m], merged[m:]                                                             # :57


def fine_matching(f0, f1, mkpts1_c, b_ids, hw0_i, hw0_f, scale1=None):
    """FineMatching.forward + get_fine_match (fine_matching.py:27-74) -> (expec_f [M, 3], mkpts1_f [M, 2]).
    kornia's spatial_expectation2d / create_meshgrid(normalized): x along the window's second axis, linspace(-1, 1, W)."""
    m, ww, c = f0.shape
    W = int(math.isqrt(ww))
    sim = torch.einsum("mc,mrc->mr", f0[:, ww // 2], f1)                                      # :43-44
    heat = torch.softmax(sim / c ** 0.5, dim=1)                                               # :45-46
    lin = torch.linspace(-1, 1, W, dtype=F64, device=f0.device)
    grid = torch.stack([lin[None, :].expand(W, W), lin[:, None].expand(W, W)], -1).reshape(ww, 2)   # :50
    coords = heat @ grid                                                                      # :49
    var = heat @ grid ** 2 - coords ** 2                                                      # :53
    std = torch.sqrt(torch.clamp(var, min=1e-10)).sum(-1)                                     # :54
    scale = hw0_i[0] / hw0_f[0]
    s1 = scale * f64(scale1, f0.device)[b_ids] if scale1 is not None else scale              # :68
    mk1 = f64(mkpts1_c, f0.device) + coords * (W // 2) * s1                                   # :69
    return torch.cat([coords, std[:, None]], -1), mk1


# ------------------------------------------------------------------------------------------------ whole hot path
def hot_path(model, feat_c0, feat_c1, feat_f0, feat_f1, hw0_i, mask0=None, mask1=None, scale0=None, scale1=None):
    """LoFTR.forward after the backbone (loftr.py:51-75) in float64, with the parameters of a loftr_b200 `model`.
    feat_c / feat_f: backbone outputs [N, C, h, w] (float64).  Returns the match keys plus conf_matrix and the
    coarse transformer outputs."""
    dev = feat_c0.device
    cfg = model.config
    n, c, h0, w0 = feat_c0.shape
    h1, w1 = feat_c1.shape[2:]
    pe = f64(model.pos_encoding.pe, dev)[0]
    x0 = (feat_c0 + pe[:, :h0, :w0]).flatten(2).transpose(1, 2)                               # loftr.py:58-59
    x1 = (feat_c1 + pe[:, :h1, :w1]).flatten(2).transpose(1, 2)
    m0 = m1 = None
    if mask0 is not None:
        mask0, mask1 = torch.as_tensor(mask0, device=dev), torch.as_tensor(mask1, device=dev)
        m0, m1 = mask0.flatten(-2), mask1.flatten(-2)
    cc = cfg["coarse"]
    x0, x1 = transformer(x0, x1, layer_weights(model.loftr_coarse, dev), cc["layer_names"], cc["nhead"], m0, m1,
                         cc.get("attention", "linear"))                                       # loftr.py:63-64
    mc = cfg["match_coarse"]
    bin_score = model.coarse_matching.bin_score if mc["match_type"] == "sinkhorn" else None
    conf = conf_matrix(x0, x1, mc, m0, m1, bin_score)
    out = coarse_match(conf, mc, hw0_i, (h0, w0), (h1, w1), mask0, mask1, scale0, scale1)    # loftr.py:67
    W = cfg["fine_window_size"]
    stride = feat_f0.shape[2] // h0
    fw = {k: f64(v, dev) for k, v in model.fine_preprocess.state_dict().items()}
    f0, f1 = fine_preprocess(feat_f0, feat_f1, x0, x1, out["b_ids"], out["i_ids"], out["j_ids"], W, stride, fw)
    if len(out["b_ids"]):
        fc = cfg["fine"]
        f0, f1 = transformer(f0, f1, layer_weights(model.loftr_fine, dev), fc["layer_names"], fc["nhead"],
                             attention=fc.get("attention", "linear"))                         # loftr.py:71-72
        out["expec_f"], out["mkpts1_f"] = fine_matching(f0, f1, out["mkpts1_c"], out["b_ids"], hw0_i,
                                                        feat_f0.shape[2:], scale1)
    else:
        out["expec_f"], out["mkpts1_f"] = torch.zeros(0, 3, dtype=F64, device=dev), out["mkpts1_c"]
    out["mkpts0_f"] = out["mkpts0_c"]
    out.update({"conf_matrix": conf, "feat_c0": x0, "feat_c1": x1})
    return out
