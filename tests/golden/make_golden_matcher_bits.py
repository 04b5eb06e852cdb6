"""Record the exact output bits of the whole matcher (tests/golden/matcher_bits.npz) for
tests/test_matcher_bits_gpu.py: the SHA-256 of every tensor output of `matcher(batch)` for each case of MATCHER_CASES, of the
live prefix of every `forward_static` output, of `lb_gemm_split` at N = 128 and 256, and of the standalone fine
transformer between windows of different sizes (FINE_TF_CASES); the outputs of FULL are stored in full as well.
Between them the cases launch every tensor-core kernel instantiation of the library (the backbone's convolutions,
every GEMM epilogue of the transformers and of both coarse matchings, the linear and full attention kernels).  A
change that only restructures kernel code must keep these bits; a change to any summation order must regenerate them
(and say so).  Needs an H100; LOFTR_B200_LIB selects the build that defines the reference bits.

    LOFTR_B200_LIB=<variant> python tests/golden/make_golden_matcher_bits.py [OUT.npz]
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from cases import CASES  # noqa: E402
from full_cases import FULL_CASES  # noqa: E402

DEV = "cuda:0"
_C = {c["name"]: c for c in CASES + FULL_CASES}
# name -> (case, path): "forward" = matcher(batch), "static" = forward_static, "conf" = forward with return_conf_matrix;
# cases with coarse_attention / fine_attention "full" run full (softmax) attention
MATCHER_CASES = {
    "ds_thr0": (_C["ds_thr0"], "forward"),
    "ds_thr0.2": (dict(_C["ds_thr0"], thr=0.2), "forward"),
    "ot_thr0": (_C["ot_thr0"], "forward"),
    "ot_prefilter": (_C["ot_prefilter"], "forward"),
    "full_ds_thr0": (_C["full_ds_thr0"], "forward"),
    "full_ot": (_C["full_ot"], "forward"),
    "masked_unequal": ({"name": "masked_unequal", "n": 2, "hw0": (128, 128), "hw1": (112, 144), "thr": 0.0,
                        "images": "rand", "valid0": [(128, 96), (104, 128)], "valid1": [(112, 128), (96, 144)],
                        "scales": True}, "forward"),
    # 128-channel layer2: the per-tap path at N = 128 (the stride-2 convolution and the 1x1 + upsample)
    "dims_128_128_256": (dict(_C["ds_thr0"], name="dims_128", n=1, block_dims=(128, 128, 256)), "forward"),
    "ds_thr0_conf": (_C["ds_thr0"], "conf"),
    "ot_masked_conf": (_C["ot_masked"], "conf"),
    "static_ds_thr0": (_C["ds_thr0"], "static"),
    "static_masked_unequal_ot": ({"name": "static_mu", "n": 2, "hw0": (128, 128), "hw1": (112, 144), "thr": 0.0,
                                  "images": "rand", "valid0": [(128, 96), (104, 128)],
                                  "valid1": [(112, 128), (96, 144)], "match_type": "sinkhorn"}, "static"),
}
GEMM_CASES = {"gemm_n128": (2, 300, 128, 256), "gemm_n256": (1, 1000, 256, 128)}   # (batches, M, N, K)
# model.loftr_fine(f0, f1[, mask0, mask1]) with the shipped ["self", "cross"] linear layers on windows of L and S rows:
# the cross layer pairs windows of different sizes.  450 windows per side: more than one window per block of the
# window kernel (at most 3 blocks per SM).  name -> (L, S, padding masks)
FINE_TF_CASES = {f"fine_tf_{l}x{s}{'_masked' if m else ''}": (l, s, m)
                 for l, s in ((25, 16), (16, 25), (32, 9)) for m in (False, True)}
FINE_TF_WINDOWS = 450
FULL = "ds_thr0"   # stored in full as well
# keys of forward_static whose first dimension is the match capacity: only the live prefix is defined
_LIST_KEYS = ("b_ids", "i_ids", "j_ids", "m_bids", "gt_mask", "mconf", "mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f",
              "expec_f")


def digest(t):
    t = t.detach().contiguous().cpu()
    return hashlib.sha256(f"{t.dtype} {tuple(t.shape)} ".encode() + t.numpy().tobytes()).hexdigest()


def _model(case, conf):
    """LoFTR with the RandomState weights of weights.py (as util.build_model), the case's attention kinds and
    block_dims; conf: return_conf_matrix."""
    import loftr_b200
    import weights as W
    from cases import build_cfg
    cfg = build_cfg(case)
    cfg["match_coarse"]["return_conf_matrix"] = conf
    cfg["resnetfpn"]["block_dims"] = list(case.get("block_dims", cfg["resnetfpn"]["block_dims"]))
    model = loftr_b200.LoFTR(cfg).eval()
    state = W.make_state({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=case.get("wseed", 0))
    if "bin_score" in case:
        state["coarse_matching.bin_score"] = np.asarray(case["bin_score"], np.float32)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    return model.to(DEV)


def matcher_outputs(name):
    """-> {key: tensor} of the matcher run of MATCHER_CASES[name] (inputs included: they must come back unchanged)."""
    from cases import build_inputs
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    case, path = MATCHER_CASES[name]
    model = _model(case, path == "conf")
    data = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in build_inputs(case).items()}
    with torch.no_grad():
        if path == "static":
            model.forward_static(data)
            m = int(data["num_matches"].item())
            data = {k: (v[:m] if k in _LIST_KEYS else v) for k, v in data.items()}
        else:
            model(data)
    torch.cuda.synchronize()
    return {k: v for k, v in data.items() if torch.is_tensor(v)}


def gemm_output(name):
    """-> lb_gemm_split(A, B) of seeded fp32 operands at GEMM_CASES[name] (B batched when there are several batches)."""
    from loftr_b200 import _lib
    from loftr_b200.loftr import _stream, split_planes
    b, m, n, k = GEMM_CASES[name]
    rs = np.random.RandomState(5)
    a = torch.from_numpy((rs.standard_normal((b * m, k)) * 3 + 1).astype(np.float32)).to(DEV)
    w = torch.from_numpy((rs.standard_normal((b * n, k)) * 3 + 1).astype(np.float32)).to(DEV)
    ah, al = split_planes(a)
    wh, wl = split_planes(w)
    out = torch.empty(b * m, n, dtype=torch.float32, device=DEV)
    lib = _lib.load()
    _lib.check(lib.lb_gemm_split(ah.data_ptr(), al.data_ptr(), k, m * k, wh.data_ptr(), wl.data_ptr(), k,
                                 n * k if b > 1 else 0, out.data_ptr(), n, m * n, b, m, n, k, _stream()))
    torch.cuda.synchronize()
    return {"out": out}


def fine_tf_output(name):
    """-> the two outputs of the fine transformer of the ds_thr0 model at FINE_TF_CASES[name] on seeded features (and
    masks that pad every window to its size after a valid prefix of at least one row)."""
    l, s, masked = FINE_TF_CASES[name]
    model = _model(_C["ds_thr0"], False)
    rs = np.random.RandomState(7)
    n = FINE_TF_WINDOWS
    f0 = torch.from_numpy(rs.standard_normal((n, l, 128)).astype(np.float32)).to(DEV)
    f1 = torch.from_numpy(rs.standard_normal((n, s, 128)).astype(np.float32)).to(DEV)
    masks = ()
    if masked:
        masks = tuple(torch.from_numpy(np.arange(rows)[None, :] < rs.randint(1, rows + 1, size=(n, 1))).to(DEV)
                      for rows in (l, s))
    g0, g1 = model.loftr_fine(f0, f1, *masks)
    torch.cuda.synchronize()
    return {"feat0": g0, "feat1": g1}


def outputs(name):
    if name in GEMM_CASES:
        return gemm_output(name)
    return fine_tf_output(name) if name in FINE_TF_CASES else matcher_outputs(name)


NAMES = list(MATCHER_CASES) + list(GEMM_CASES) + list(FINE_TF_CASES)


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "matcher_bits.npz")
    out = {}
    for name in NAMES:
        res = outputs(name)
        out[f"keys_{name}"] = np.array(sorted(res))
        for k, v in res.items():
            out[f"sha_{name}_{k}"] = np.array(digest(v))
            if name == FULL:
                out[f"full_{name}_{k}"] = v.cpu().numpy()
        print(name, {k: len(v) for k, v in res.items() if v.dim()}, flush=True)
    np.savez_compressed(out_path, **out)
    print(f"-> {out_path} ({os.path.getsize(out_path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
