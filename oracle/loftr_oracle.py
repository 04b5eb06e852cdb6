"""CPU oracle for the LoFTR matching hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A numpy (float32) restatement of the reference algorithm (zju3dv/LoFTR; file:line citations are
relative to the reference root) for every stage the CUDA engine replaces.  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may import it; the
product package `loftr_b200` never does.

Pinning: the reference ships no golden vectors (SURVEY.md §4), so this oracle is pinned against
outputs of the reference itself, run in the authoring container by `tests/golden/make_golden.py`
(fixtures under `tests/golden/*.npz`, checked by `tests/test_oracle_golden.py`).

All arrays are numpy float32 unless noted; shapes follow the reference docstrings.
"""
from __future__ import annotations

import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

F32 = np.float32
INF = 1e9  # coarse_matching.py:6

# numpy ufuncs release the GIL, so the big elementwise passes (softmax over L x S, LayerNorm, elu) are
# row-blocked over a thread pool -- the reference's torch-CPU kernels use every host core too, and this
# port is also the timed CPU baseline (bench.py).  Dense products go through BLAS (`@`).
_POOL = ThreadPoolExecutor(max_workers=min(os.cpu_count() or 1, int(os.environ.get("LOFTR_ORACLE_THREADS", "32"))))


def _blocked(fn, n_rows, min_rows=64):
    """Run fn(lo, hi) over row blocks [lo, hi) of an array with n_rows leading rows, in parallel."""
    workers = _POOL._max_workers
    if n_rows < 2 * min_rows or workers == 1:
        fn(0, n_rows)
        return
    step = max(min_rows, -(-n_rows // (workers * 2)))
    list(_POOL.map(lambda lo: fn(lo, min(lo + step, n_rows)), range(0, n_rows, step)))


# --------------------------------------------------------------------------------------------------
# position encoding  (src/loftr/utils/position_encoding.py:11-42)
# --------------------------------------------------------------------------------------------------
def position_encoding_sine(d_model: int, h: int, w: int, temp_bug_fix: bool = True) -> np.ndarray:
    """pe[:, :h, :w] of PositionEncodingSine -> [d_model, h, w] float32."""
    y_position = np.arange(1, h + 1, dtype=F32)[:, None] * np.ones((1, w), F32)  # cumsum of ones, :23
    x_position = np.ones((h, 1), F32) * np.arange(1, w + 1, dtype=F32)[None, :]  # :24
    k = np.arange(0, d_model // 2, 2, dtype=F32)
    if temp_bug_fix:
        div_term = np.exp(k * F32(-math.log(10000.0) / (d_model // 2))).astype(F32)  # :26
    else:  # python precedence of the buggy variant: (-log(1e4) / d_model) // 2     # :28
        div_term = np.exp(k * F32(-math.log(10000.0) / d_model // 2)).astype(F32)
    div_term = div_term[:, None, None]
    pe = np.zeros((d_model, h, w), F32)
    pe[0::4] = np.sin(x_position[None] * div_term)
    pe[1::4] = np.cos(x_position[None] * div_term)
    pe[2::4] = np.sin(y_position[None] * div_term)
    pe[3::4] = np.cos(y_position[None] * div_term)
    return pe


def coarse_tokens(feat_c: np.ndarray, pe: np.ndarray) -> np.ndarray:
    """pos_encoding + rearrange 'n c h w -> n (h w) c'  (src/loftr/loftr.py:58-59)."""
    n, c, h, w = feat_c.shape
    x = feat_c + pe[None, :, :h, :w]
    return np.ascontiguousarray(x.reshape(n, c, h * w).transpose(0, 2, 1))


# --------------------------------------------------------------------------------------------------
# linear attention + encoder layer + transformer
# --------------------------------------------------------------------------------------------------
def _elu_feature_map(x: np.ndarray) -> np.ndarray:
    """elu(x) + 1  (linear_attention.py:10-11)."""
    out = np.empty(x.shape, F32)
    x2, o2 = x.reshape(-1, x.shape[-1]), out.reshape(-1, x.shape[-1])

    def body(lo, hi):
        xb = x2[lo:hi]
        o2[lo:hi] = np.where(xb > 0, xb, np.expm1(np.minimum(xb, 0))) + F32(1)

    _blocked(body, x2.shape[0], 512)
    return out


def linear_attention(q, k, v, q_mask=None, kv_mask=None, eps=1e-6):
    """LinearAttention.forward (linear_attention.py:20-47).  q [N,L,H,D], k/v [N,S,H,D]."""
    Q = _elu_feature_map(q)
    K = _elu_feature_map(k)
    if q_mask is not None:
        Q = Q * q_mask[:, :, None, None].astype(F32)
    if kv_mask is not None:
        K = K * kv_mask[:, :, None, None].astype(F32)
        v = v * kv_mask[:, :, None, None].astype(F32)
    v_length = v.shape[1]
    v = v / F32(v_length)                                       # :41-42
    Kt = K.transpose(0, 2, 3, 1)                                # [N,H,D,S]
    KV = Kt @ v.transpose(0, 2, 1, 3)                           # einsum nshd,nshv->nhdv            :43
    Qh = Q.transpose(0, 2, 1, 3)                                # [N,H,L,D]
    Z = F32(1) / ((Qh @ K.sum(axis=1)[:, :, :, None])[..., 0] + F32(eps))   # einsum nlhd,nhd->nlh  :44
    out = (Qh @ KV) * Z[..., None] * F32(v_length)              # einsum nlhd,nhdv,nlh->nlhv        :45
    return np.ascontiguousarray(out.transpose(0, 2, 1, 3)).astype(F32)


def full_attention(q, k, v, q_mask=None, kv_mask=None):
    """FullAttention.forward (linear_attention.py:56-81), dropout off.  q [N,L,H,D], k/v [N,S,H,D] -> [N,L,H,D].
    A = softmax(Q K^T / sqrt(D)) over s with -inf logits where !(q_mask[l] & kv_mask[s]); values are not masked.
    Row-blocked so that L x S x H never exists at once.

    Masked rows: the reference gives every logit of a padded query row -inf, so its softmax (and, through the values
    of the next layer, every row after it) is NaN.  The engine and this oracle give such a row, and a row without any
    valid key, a zero message instead; valid rows equal the reference wherever it is finite."""
    n, L, H, D = q.shape
    qh = np.ascontiguousarray(q.transpose(0, 2, 1, 3)).astype(F32)          # [N,H,L,D]
    kh = np.ascontiguousarray(k.transpose(0, 2, 3, 1)).astype(F32)          # [N,H,D,S]
    vh = np.ascontiguousarray(v.transpose(0, 2, 1, 3)).astype(F32)          # [N,H,S,D]
    temp = F32(1.0 / D ** 0.5)                                              # :77
    out = np.zeros((n, H, L, D), F32)
    for b in range(n):
        kbias = None
        if kv_mask is not None:
            kbias = np.where(np.asarray(kv_mask[b]).astype(bool), F32(0), F32(-np.inf)).astype(F32)

        def body(lo, hi, b=b, kbias=kbias):
            qk = qh[b, :, lo:hi] @ kh[b]                                     # einsum nlhd,nshd->nlsh  :70
            if kbias is not None:
                qk = qk + kbias[None, None, :]                               # masked_fill(-inf)  :72-73
            z = temp * qk
            m = z.max(axis=-1, keepdims=True)
            m = np.where(np.isfinite(m), m, F32(0))
            e = np.exp(z - m)
            ssum = e.sum(axis=-1, keepdims=True)
            a = np.where(ssum > 0, e / np.where(ssum > 0, ssum, F32(1)), F32(0))   # softmax(dim=2)  :78
            o = a @ vh[b]                                                    # einsum nlsh,nshd->nlhd  :81
            if q_mask is not None:
                o = o * np.asarray(q_mask[b, lo:hi]).astype(F32)[None, :, None]
            out[b, :, lo:hi] = o

        _blocked(body, L, 256)
    return np.ascontiguousarray(out.transpose(0, 2, 1, 3)).astype(F32)


ATTENTION = {"linear": linear_attention, "full": full_attention}   # transformer.py:21


def layer_norm(x, g, b, eps=1e-5):
    """nn.LayerNorm over the last axis (biased variance), float32."""
    out = np.empty(x.shape, F32)
    x2, o2 = x.reshape(-1, x.shape[-1]), out.reshape(-1, x.shape[-1])

    def body(lo, hi):
        xb = x2[lo:hi]
        mu = xb.mean(axis=-1, keepdims=True, dtype=F32)
        d = xb - mu
        var = (d * d).mean(axis=-1, keepdims=True, dtype=F32)
        o2[lo:hi] = d / np.sqrt(var + F32(eps)) * g + b

    _blocked(body, x2.shape[0], 512)
    return out


def encoder_layer(x, source, w, nhead, x_mask=None, source_mask=None, attention="linear"):
    """LoFTREncoderLayer.forward (transformer.py:35-58) with attention 'linear' or 'full'.  `w` maps the layer's
    state_dict suffixes ('q_proj.weight', ..., 'norm2.bias') to arrays ([out, in] for Linear)."""
    bs, _, c = x.shape
    dim = c // nhead
    q = (x @ w["q_proj.weight"].T).reshape(bs, -1, nhead, dim)          # :47
    k = (source @ w["k_proj.weight"].T).reshape(bs, -1, nhead, dim)     # :48
    v = (source @ w["v_proj.weight"].T).reshape(bs, -1, nhead, dim)     # :49
    msg = ATTENTION[attention](q, k, v, x_mask, source_mask)            # :50
    msg = msg.reshape(bs, -1, nhead * dim) @ w["merge.weight"].T        # :51
    msg = layer_norm(msg, w["norm1.weight"], w["norm1.bias"])           # :52
    h = np.concatenate([x, msg], axis=2) @ w["mlp.0.weight"].T          # :55
    h = np.maximum(h, 0)
    msg = h @ w["mlp.2.weight"].T
    msg = layer_norm(msg, w["norm2.weight"], w["norm2.bias"])           # :56
    return (x + msg).astype(F32)                                        # :58


def local_feature_transformer(feat0, feat1, layers, layer_names, nhead, mask0=None, mask1=None, attention="linear"):
    """LocalFeatureTransformer.forward (transformer.py:80-101): interleaved self / cross layers, one attention kind
    for every layer; in a cross layer feat1 attends to the already updated feat0 (:96-97)."""
    a = attention
    for w, name in zip(layers, layer_names):
        if name == "self":
            feat0 = encoder_layer(feat0, feat0, w, nhead, mask0, mask0, a)
            feat1 = encoder_layer(feat1, feat1, w, nhead, mask1, mask1, a)
        elif name == "cross":
            feat0 = encoder_layer(feat0, feat1, w, nhead, mask0, mask1, a)
            feat1 = encoder_layer(feat1, feat0, w, nhead, mask1, mask0, a)
        else:
            raise KeyError(name)
    return feat0, feat1


# --------------------------------------------------------------------------------------------------
# coarse matching
# --------------------------------------------------------------------------------------------------
def _logsumexp(x, axis):
    m = x.max(axis=axis, keepdims=True)
    return (m + np.log(np.exp(x - m).sum(axis=axis, keepdims=True))).squeeze(axis)


def _softmax(x, axis):
    """softmax along `axis` of a 2-D or 3-D float32 array (threaded over the other axes)."""
    if x.ndim == 2:
        return _softmax(x[None], axis + 1)[0]
    out = np.empty(x.shape, F32)
    if axis == 2:
        x2, o2 = x.reshape(-1, x.shape[2]), out.reshape(-1, x.shape[2])

        def body(lo, hi):
            xb = x2[lo:hi]
            e = np.exp(xb - xb.max(axis=1, keepdims=True))
            o2[lo:hi] = e / e.sum(axis=1, keepdims=True)

        _blocked(body, x2.shape[0])
    elif axis == 1:
        def body(lo, hi):  # column blocks
            xb = x[:, :, lo:hi]
            e = np.exp(xb - xb.max(axis=1, keepdims=True))
            out[:, :, lo:hi] = e / e.sum(axis=1, keepdims=True)

        _blocked(body, x.shape[2])
    else:
        raise ValueError(axis)
    return out


def log_optimal_transport(scores, alpha, iters):
    """log_optimal_transport / log_sinkhorn_iterations (third_party/SuperGluePretrainedNetwork/
    models/superglue.py:141-170), restated from the formulas; returns [b, m+1, n+1]."""
    b, m, n = scores.shape
    alpha = F32(alpha)
    couplings = np.full((b, m + 1, n + 1), alpha, F32)       # dustbin row / column / corner  :156-160
    couplings[:, :m, :n] = scores
    norm = F32(-math.log(m + n))                             # :162
    log_mu = np.concatenate([np.full(m, norm, F32), np.array([math.log(n) + norm], F32)])  # :163
    log_nu = np.concatenate([np.full(n, norm, F32), np.array([math.log(m) + norm], F32)])  # :164
    u = np.zeros((b, m + 1), F32)
    v = np.zeros((b, n + 1), F32)
    for _ in range(iters):                                   # :144-148
        u = log_mu[None] - _logsumexp(couplings + v[:, None, :], axis=2)
        v = log_nu[None] - _logsumexp(couplings + u[:, :, None], axis=1)
    return (couplings + u[:, :, None] + v[:, None, :] - norm).astype(F32)   # :148,169


def _mask_border(mask5, b):
    """mask_border (coarse_matching.py:8-25) on a bool [N,H0,W0,H1,W1] array, in place."""
    if b <= 0:
        return
    mask5[:, :b] = False
    mask5[:, :, :b] = False
    mask5[:, :, :, :b] = False
    mask5[:, :, :, :, :b] = False
    mask5[:, -b:] = False
    mask5[:, :, -b:] = False
    mask5[:, :, :, -b:] = False
    mask5[:, :, :, :, -b:] = False


def _mask_border_with_padding(mask5, bd, p_m0, p_m1):
    """mask_border_with_padding (coarse_matching.py:28-43)."""
    if bd <= 0:
        return
    mask5[:, :bd] = False
    mask5[:, :, :bd] = False
    mask5[:, :, :, :bd] = False
    mask5[:, :, :, :, :bd] = False
    h0s, w0s = p_m0.sum(1).max(-1).astype(int), p_m0.sum(-1).max(-1).astype(int)
    h1s, w1s = p_m1.sum(1).max(-1).astype(int), p_m1.sum(-1).max(-1).astype(int)
    for b_idx, (h0, w0, h1, w1) in enumerate(zip(h0s, w0s, h1s, w1s)):
        mask5[b_idx, h0 - bd:] = False
        mask5[b_idx, :, w0 - bd:] = False
        mask5[b_idx, :, :, h1 - bd:] = False
        mask5[b_idx, :, :, :, w1 - bd:] = False


def coarse_conf_matrix(feat_c0, feat_c1, cfg, mask_c0=None, mask_c1=None, bin_score=None):
    """CoarseMatching.forward up to conf_matrix (coarse_matching.py:103-143).  masks: bool [N,L],[N,S]."""
    c = feat_c0.shape[-1]
    f0 = feat_c0 / F32(c ** 0.5)
    f1 = feat_c1 / F32(c ** 0.5)
    pad = None
    if mask_c0 is not None:
        pad = ~(mask_c0[..., None] & mask_c1[:, None])
    if cfg["match_type"] == "dual_softmax":
        sim = (f0 @ f1.transpose(0, 2, 1)) / F32(cfg["dsmax_temperature"])         # einsum nlc,nsc->nls  :109-110
        if pad is not None:
            sim[pad] = -INF                                                        # :111-114
        conf = _softmax(sim, 1) * _softmax(sim, 2)                                 # :115
        return conf.astype(F32), None
    if cfg["match_type"] == "sinkhorn":
        sim = f0 @ f1.transpose(0, 2, 1)                                           # einsum nlc,nsc->nls  :119
        if pad is not None:
            sim[pad] = -INF
        log_assign = log_optimal_transport(sim, bin_score, cfg["skh_iters"])      # :126-127
        assign = np.exp(log_assign)
        conf = assign[:, :-1, :-1].copy()
        if cfg.get("skh_prefilter", False):                                        # :132-136
            L, S = conf.shape[1], conf.shape[2]
            filter0 = (assign.argmax(axis=2) == S)[:, :-1]
            filter1 = (assign.argmax(axis=1) == L)[:, :-1]
            conf[np.broadcast_to(filter0[..., None], conf.shape)] = 0
            conf[np.broadcast_to(filter1[:, None], conf.shape)] = 0
        return conf.astype(F32), assign.astype(F32)
    raise NotImplementedError(cfg["match_type"])


def get_coarse_match(conf, cfg, hw0_i, hw0_c, hw1_c, mask0=None, mask1=None, scale0=None, scale1=None):
    """CoarseMatching.get_coarse_match, eval path (coarse_matching.py:150-197,238-261).
    mask0/mask1: bool [N,h0c,w0c] / [N,h1c,w1c].  Returns the dict of coarse matches (int64 ids)."""
    n = conf.shape[0]
    h0c, w0c = hw0_c
    h1c, w1c = hw1_c
    mask = conf > F32(cfg["thr"])                                                  # :167
    mask5 = mask.reshape(n, h0c, w0c, h1c, w1c).copy()
    if mask0 is None:
        _mask_border(mask5, cfg["border_rm"])                                      # :170-171
    else:
        _mask_border_with_padding(mask5, cfg["border_rm"], mask0, mask1)           # :172-174
    mask = mask5.reshape(conf.shape)
    mask = mask & (conf == conf.max(axis=2, keepdims=True)) & (conf == conf.max(axis=1, keepdims=True))  # :179-181
    mask_v = mask.max(axis=2)                                                      # :185
    all_j = mask.argmax(axis=2)
    b_ids, i_ids = np.nonzero(mask_v)                                              # :186
    j_ids = all_j[b_ids, i_ids]
    mconf = conf[b_ids, i_ids, j_ids]
    scale = hw0_i[0] / hw0_c[0]                                                    # :241
    s0 = F32(scale) * scale0[b_ids].astype(F32) if scale0 is not None else F32(scale)
    s1 = F32(scale) * scale1[b_ids].astype(F32) if scale1 is not None else F32(scale)
    mkpts0_c = (np.stack([i_ids % w0c, i_ids // w0c], axis=1).astype(F32) * s0).astype(F32)   # :244-246
    mkpts1_c = (np.stack([j_ids % w1c, j_ids // w1c], axis=1).astype(F32) * s1).astype(F32)   # :247-249
    keep = mconf != 0                                                              # :253-258
    return {
        "b_ids": b_ids.astype(np.int64), "i_ids": i_ids.astype(np.int64), "j_ids": j_ids.astype(np.int64),
        "gt_mask": mconf == 0, "m_bids": b_ids[keep].astype(np.int64),
        "mkpts0_c": mkpts0_c[keep], "mkpts1_c": mkpts1_c[keep], "mconf": mconf[keep].astype(F32),
    }


def coarse_matching(feat_c0, feat_c1, cfg, hw0_i, hw0_c, hw1_c, mask0=None, mask1=None, scale0=None,
                    scale1=None, bin_score=None):
    """CoarseMatching.forward (coarse_matching.py:87-148).  mask0/mask1 are the [N,h,w] grids."""
    m0 = mask0.reshape(mask0.shape[0], -1) if mask0 is not None else None
    m1 = mask1.reshape(mask1.shape[0], -1) if mask1 is not None else None
    conf, assign = coarse_conf_matrix(feat_c0, feat_c1, cfg, m0, m1, bin_score)
    out = get_coarse_match(conf, cfg, hw0_i, hw0_c, hw1_c, mask0, mask1, scale0, scale1)
    out["conf_matrix"] = conf
    return out


# --------------------------------------------------------------------------------------------------
# fine level
# --------------------------------------------------------------------------------------------------
def gather_windows(feat_f, b_ids, idx, wc, W, stride):
    """F.unfold(kernel=W, stride, padding=W//2) + rearrange + [b_ids, idx] (fine_preprocess.py:40-47),
    restated as a direct gather (SURVEY.md §9 V4): win[m, ky*W+kx, c] =
    feat_f[b, c, stride*y - W//2 + ky, stride*x - W//2 + kx], zero outside.  feat_f: [N, C, Hf, Wf]."""
    n, c, hf, wf = feat_f.shape
    m = len(b_ids)
    out = np.zeros((m, W * W, c), F32)
    cy, cx = idx // wc, idx % wc
    for ky in range(W):
        for kx in range(W):
            y = stride * cy - W // 2 + ky
            x = stride * cx - W // 2 + kx
            ok = (y >= 0) & (y < hf) & (x >= 0) & (x < wf)
            vals = feat_f[b_ids[ok], :, y[ok], x[ok]]
            out[ok, ky * W + kx, :] = vals
    return out


def fine_preprocess(feat_f0, feat_f1, feat_c0, feat_c1, b_ids, i_ids, j_ids, w0c, w1c, W, stride, w):
    """FinePreprocess.forward with fine_concat_coarse_feat=True (fine_preprocess.py:29-59).
    `w`: 'down_proj.weight/bias', 'merge_feat.weight/bias'."""
    cf = feat_f0.shape[1]
    if len(b_ids) == 0:
        return np.zeros((0, W * W, cf), F32), np.zeros((0, W * W, cf), F32)
    win0 = gather_windows(feat_f0, b_ids, i_ids, w0c, W, stride)
    win1 = gather_windows(feat_f1, b_ids, j_ids, w1c, W, stride)
    fc = np.concatenate([feat_c0[b_ids, i_ids], feat_c1[b_ids, j_ids]], 0)            # :50-51
    c_win = fc @ w["down_proj.weight"].T + w["down_proj.bias"]                        # [2M, cf]
    cat = np.concatenate([np.concatenate([win0, win1], 0),
                          np.repeat(c_win[:, None, :], W * W, axis=1)], -1)          # :52-55
    merged = cat @ w["merge_feat.weight"].T + w["merge_feat.bias"]
    m = len(b_ids)
    return merged[:m].astype(F32), merged[m:].astype(F32)                             # :56


def fine_matching(f0, f1, mkpts0_c, mkpts1_c, b_ids, hw0_i, hw0_f, scale1=None):
    """FineMatching.forward + get_fine_match (fine_matching.py:15-74).  f0/f1: [M, WW, C].
    kornia's spatial_expectation2d(normalized) / create_meshgrid(normalized) are restated as the
    expectation over the grid linspace(-1, 1, W)^2 with x along the window's second axis."""
    m, ww, c = f0.shape
    W = int(math.sqrt(ww))
    scale = hw0_i[0] / hw0_f[0]
    if m == 0:                                                                        # :33-41
        return {"expec_f": np.zeros((0, 3), F32), "mkpts0_f": mkpts0_c, "mkpts1_f": mkpts1_c}
    picked = f0[:, ww // 2, :]                                                        # :43
    sim = (f1 @ picked[:, :, None])[..., 0]                                           # einsum mc,mrc->mr  :44
    heat = _softmax(F32(1.0 / c ** 0.5) * sim, 1)                                     # :45-46
    lin = np.linspace(-1, 1, W).astype(F32)
    gx = np.tile(lin[None, :], (W, 1)).reshape(-1)
    gy = np.tile(lin[:, None], (1, W)).reshape(-1)
    grid = np.stack([gx, gy], -1)                                                     # [WW, 2]  :50
    coords = heat @ grid                                                              # [M, 2]   :49
    var = (heat[:, :, None] * grid[None] ** 2).sum(1) - coords ** 2                   # :53
    std = np.sqrt(np.clip(var, 1e-10, None)).sum(-1)                                  # :54
    expec = np.concatenate([coords, std[:, None]], -1).astype(F32)                    # :57
    s1 = F32(scale) * scale1[b_ids].astype(F32) if scale1 is not None else F32(scale)  # :68
    mk1 = mkpts1_c + (coords * F32(W // 2) * s1)[: len(mkpts1_c)]                      # :69
    return {"expec_f": expec, "mkpts0_f": mkpts0_c, "mkpts1_f": mk1.astype(F32)}


# --------------------------------------------------------------------------------------------------
# whole hot path (LoFTR.forward after the backbone, loftr.py:51-75)
# --------------------------------------------------------------------------------------------------
def split_layers(state, prefix, n_layers):
    """state_dict (name -> array) -> list of per-layer weight dicts for `prefix`.layers.{i}."""
    names = ["q_proj.weight", "k_proj.weight", "v_proj.weight", "merge.weight", "mlp.0.weight", "mlp.2.weight",
             "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias"]
    return [{k: state[f"{prefix}.layers.{i}.{k}"] for k in names} for i in range(n_layers)]


def hot_path(feat_c0, feat_c1, feat_f0, feat_f1, state, cfg, hw0_i, hw1_i, mask0=None, mask1=None, scale0=None,
             scale1=None):
    """Backbone outputs (NCHW) -> every key LoFTR.forward writes after the backbone.  `cfg` is the
    reference's lower-case config dict (cfg['coarse' | 'fine']['attention']: 'linear' when absent); `state` the
    state_dict as numpy arrays."""
    n = feat_c0.shape[0]
    hw0_c, hw1_c = feat_c0.shape[2:], feat_c1.shape[2:]
    hw0_f, hw1_f = feat_f0.shape[2:], feat_f1.shape[2:]
    cc = cfg["coarse"]
    pe = position_encoding_sine(cc["d_model"], max(hw0_c[0], hw1_c[0]), max(hw0_c[1], hw1_c[1]),
                                cc.get("temp_bug_fix", True))
    x0, x1 = coarse_tokens(feat_c0, pe), coarse_tokens(feat_c1, pe)
    m0 = mask0.reshape(n, -1) if mask0 is not None else None
    m1 = mask1.reshape(n, -1) if mask1 is not None else None
    layers = split_layers(state, "loftr_coarse", len(cc["layer_names"]))
    x0, x1 = local_feature_transformer(x0, x1, layers, cc["layer_names"], cc["nhead"], m0, m1,
                                       cc.get("attention", "linear"))
    mc = cfg["match_coarse"]
    bin_score = state.get("coarse_matching.bin_score")
    out = coarse_matching(x0, x1, mc, hw0_i, hw0_c, hw1_c, mask0, mask1, scale0, scale1, bin_score)
    W = cfg["fine_window_size"]
    stride = hw0_f[0] // hw0_c[0]
    fw = {k: state[f"fine_preprocess.{k}"] for k in
          ["down_proj.weight", "down_proj.bias", "merge_feat.weight", "merge_feat.bias"]}
    f0, f1 = fine_preprocess(feat_f0, feat_f1, x0, x1, out["b_ids"], out["i_ids"], out["j_ids"], hw0_c[1],
                             hw1_c[1], W, stride, fw)
    if f0.shape[0] != 0:
        fc = cfg["fine"]
        flayers = split_layers(state, "loftr_fine", len(fc["layer_names"]))
        f0, f1 = local_feature_transformer(f0, f1, flayers, fc["layer_names"], fc["nhead"],
                                           attention=fc.get("attention", "linear"))
    out.update(fine_matching(f0, f1, out["mkpts0_c"], out["mkpts1_c"], out["b_ids"], hw0_i, hw0_f, scale1))
    out.update({"feat_c0": x0, "feat_c1": x1, "feat_f0_unfold": f0, "feat_f1_unfold": f1,
                "hw0_c": tuple(hw0_c), "hw1_c": tuple(hw1_c), "hw0_f": tuple(hw0_f), "hw1_f": tuple(hw1_f)})
    return out
