"""CPU oracle of full (softmax) attention -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A numpy (float32) restatement of the reference's `FullAttention` (src/loftr/loftr_module/linear_attention.py:50-81)
and of the encoder / transformer / hot path with an `attention` argument per transformer ('linear' | 'full',
transformer.py:21).  Everything else is the shared oracle (oracle/loftr_oracle.py); this module only adds the
attention choice on top of it.  Pinned against the reference by the FULL_CASES goldens (tests/golden/full_cases.py).

Masked rows: the reference gives every logit of a padded query row -inf, so its softmax (and, through the values of
the next layer, every row after it) is NaN.  The engine and this oracle give such a row, and a row without any valid
key, a zero message instead; valid rows equal the reference wherever it is finite.
"""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np
import torch

import util
import weights as W
from cases import build_inputs
from full_cases import build_full_cfg
from oracle import loftr_oracle as O

F32 = np.float32


def full_attention(q, k, v, q_mask=None, kv_mask=None):
    """FullAttention.forward (linear_attention.py:56-81), dropout off.  q [N,L,H,D], k/v [N,S,H,D] -> [N,L,H,D].
    A = softmax(Q K^T / sqrt(D)) over s with -inf logits where !(q_mask[l] & kv_mask[s]); values are not masked.
    Row-blocked so that L x S x H never exists at once."""
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

        O._blocked(body, L, 256)
    return np.ascontiguousarray(out.transpose(0, 2, 1, 3)).astype(F32)


def encoder_layer(x, source, w, nhead, x_mask=None, source_mask=None, attention="linear"):
    """LoFTREncoderLayer.forward (transformer.py:35-58) with the attention kind of transformer.py:21."""
    if attention == "linear":
        return O.encoder_layer(x, source, w, nhead, x_mask, source_mask)
    if attention != "full":
        raise ValueError(attention)
    bs, _, c = x.shape
    dim = c // nhead
    q = (x @ w["q_proj.weight"].T).reshape(bs, -1, nhead, dim)          # :47
    k = (source @ w["k_proj.weight"].T).reshape(bs, -1, nhead, dim)     # :48
    v = (source @ w["v_proj.weight"].T).reshape(bs, -1, nhead, dim)     # :49
    msg = full_attention(q, k, v, x_mask, source_mask)                  # :50
    msg = msg.reshape(bs, -1, nhead * dim) @ w["merge.weight"].T        # :51
    msg = O.layer_norm(msg, w["norm1.weight"], w["norm1.bias"])         # :52
    h = np.concatenate([x, msg], axis=2) @ w["mlp.0.weight"].T          # :55
    h = np.maximum(h, 0)
    msg = h @ w["mlp.2.weight"].T
    msg = O.layer_norm(msg, w["norm2.weight"], w["norm2.bias"])         # :56
    return (x + msg).astype(F32)                                        # :58


def local_feature_transformer(feat0, feat1, layers, layer_names, nhead, mask0=None, mask1=None, attention="linear"):
    """LocalFeatureTransformer.forward (transformer.py:80-101) with one attention kind for every layer."""
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


def hot_path(feat_c0, feat_c1, feat_f0, feat_f1, state, cfg, hw0_i, hw1_i, mask0=None, mask1=None, scale0=None,
             scale1=None, attention=None):
    """oracle.hot_path with the transformers' attention kinds: attention = (coarse, fine); None reads
    cfg['coarse' | 'fine']['attention'] ('linear' when absent)."""
    if attention is None:
        attention = (cfg["coarse"].get("attention", "linear"), cfg["fine"].get("attention", "linear"))
    n = feat_c0.shape[0]
    hw0_c, hw1_c = feat_c0.shape[2:], feat_c1.shape[2:]
    hw0_f = feat_f0.shape[2:]
    cc = cfg["coarse"]
    pe = O.position_encoding_sine(cc["d_model"], max(hw0_c[0], hw1_c[0]), max(hw0_c[1], hw1_c[1]),
                                  cc.get("temp_bug_fix", True))
    x0, x1 = O.coarse_tokens(feat_c0, pe), O.coarse_tokens(feat_c1, pe)
    m0 = mask0.reshape(n, -1) if mask0 is not None else None
    m1 = mask1.reshape(n, -1) if mask1 is not None else None
    layers = O.split_layers(state, "loftr_coarse", len(cc["layer_names"]))
    x0, x1 = local_feature_transformer(x0, x1, layers, cc["layer_names"], cc["nhead"], m0, m1, attention[0])
    bin_score = state.get("coarse_matching.bin_score")
    out = O.coarse_matching(x0, x1, cfg["match_coarse"], hw0_i, hw0_c, hw1_c, mask0, mask1, scale0, scale1, bin_score)
    W = cfg["fine_window_size"]
    stride = hw0_f[0] // hw0_c[0]
    fw = {k: state[f"fine_preprocess.{k}"] for k in
          ["down_proj.weight", "down_proj.bias", "merge_feat.weight", "merge_feat.bias"]}
    f0, f1 = O.fine_preprocess(feat_f0, feat_f1, x0, x1, out["b_ids"], out["i_ids"], out["j_ids"], hw0_c[1],
                               hw1_c[1], W, stride, fw)
    if f0.shape[0] != 0:
        fc = cfg["fine"]
        flayers = O.split_layers(state, "loftr_fine", len(fc["layer_names"]))
        f0, f1 = local_feature_transformer(f0, f1, flayers, fc["layer_names"], fc["nhead"], attention=attention[1])
    out.update(O.fine_matching(f0, f1, out["mkpts0_c"], out["mkpts1_c"], out["b_ids"], hw0_i, hw0_f, scale1))
    out.update({"feat_c0": x0, "feat_c1": x1, "feat_f0_unfold": f0, "feat_f1_unfold": f1,
                "hw0_c": tuple(hw0_c), "hw1_c": tuple(hw1_c), "hw0_f": tuple(hw0_f),
                "hw1_f": tuple(feat_f1.shape[2:])})
    return out


def _build_model(case):
    """loftr_b200.LoFTR (CPU) with the case's attention kinds and the deterministic weights of tests/golden/weights.py."""
    import loftr_b200
    cfg = build_full_cfg(case)
    model = loftr_b200.LoFTR(cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    state = W.make_state(shapes, seed=case.get("wseed", 0))
    model.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    return model, cfg, state


def _forward_per_pair(case):
    """PyTorch backbone, then hot_path one pair at a time, + fp64 near-tie statistics of every pair (dual-softmax)."""
    model, cfg, state = _build_model(case)
    inp = build_inputs(case)
    keys = ["b_ids", "i_ids", "j_ids", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f"]
    parts = {k: [] for k in keys}
    rows, cols = [], []
    opt = lambda name, b: inp[name][b:b + 1] if name in inp else None
    for b in range(case["n"]):
        with torch.no_grad():
            i0, i1 = torch.from_numpy(inp["image0"][b:b + 1]), torch.from_numpy(inp["image1"][b:b + 1])
            if i0.shape == i1.shape:
                fc, ff = model.backbone(torch.cat([i0, i1], 0))
                (c0, c1), (f0, f1) = fc.split(1), ff.split(1)
            else:
                (c0, f0), (c1, f1) = model.backbone(i0), model.backbone(i1)
        c0, c1, f0, f1 = (t.numpy() for t in (c0, c1, f0, f1))
        out = hot_path(c0, c1, f0, f1, state, cfg, inp["image0"].shape[2:], inp["image1"].shape[2:],
                       opt("mask0", b), opt("mask1", b), opt("scale0", b), opt("scale1", b))
        for k in keys:
            parts[k].append(out[k] + b if k == "b_ids" else out[k])
        if cfg["match_coarse"]["match_type"] == "dual_softmax":
            m0 = inp["mask0"][b].reshape(-1) if "mask0" in inp else None
            m1 = inp["mask1"][b].reshape(-1) if "mask1" in inp else None
            r, c = util.near_tie_top2_f64(out["feat_c0"][0], out["feat_c1"][0], cfg["match_coarse"], m0, m1)
            rows.append(r)
            cols.append(c)
    res = {k: np.concatenate(v, 0) for k, v in parts.items()}
    gold = {"row_top2_f64": np.stack(rows), "col_top2_f64": np.stack(cols)} if rows else None
    return res, gold


def oracle_forward_per_pair(case, use_cache=True):
    """Cached `_forward_per_pair`, like util.oracle_forward_per_pair: entries live in the git-ignored
    tests/_oracle_cache/ under a hash of the case and of every source the result depends on (missing / stale entries
    are recomputed); tools/precompute_oracle.py fills them on a CPU machine."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    h = hashlib.sha1(json.dumps(case, sort_keys=True, default=str).encode())
    for rel in ("oracle/loftr_oracle.py", "tests/full_oracle.py", "tests/util.py", "tests/golden/weights.py",
                "tests/golden/cases.py", "tests/golden/full_cases.py", "loftr_b200/backbone.py", "loftr_b200/config.py"):
        h.update(open(os.path.join(root, rel), "rb").read())
    path = os.path.join(util.CACHE, f"{case['name']}_{h.hexdigest()[:20]}.npz")
    if use_cache and os.path.exists(path):
        z = dict(np.load(path))
        gold = {k: z.pop(k) for k in ("row_top2_f64", "col_top2_f64") if k in z} or None
        return z, gold
    res, gold = _forward_per_pair(case)
    if use_cache:
        try:
            os.makedirs(util.CACHE, exist_ok=True)
            np.savez(path + ".tmp.npz", **res, **(gold or {}))
            os.replace(path + ".tmp.npz", path)
        except OSError:
            pass
    return res, gold
