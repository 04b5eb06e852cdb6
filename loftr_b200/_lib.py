"""ctypes binding of the C ABI declared in include/loftr_b200.h.

The CUDA library is mandatory: there is no PyTorch / CPU fallback for the hot path.  Importing this
module on a machine where the library has not been built raises immediately; calling a compute entry
point without an sm_90 (H100) device fails inside the library with a clear message.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# LOFTR_B200_LIB selects another build of the library under lib/ (e.g. "base" -> libloftr_b200_base.so), so that two
# builds can be compared in the same tree
_VARIANT = os.environ.get("LOFTR_B200_LIB", "")
LIB_PATH = os.path.join(_HERE, "lib", f"libloftr_b200{'_' + _VARIANT if _VARIANT else ''}.so")

MATCH_DUAL_SOFTMAX = 0
MATCH_SINKHORN = 1
LAYER_SELF = 0
LAYER_CROSS = 1
LAYER_SELF_FULL = 2
LAYER_CROSS_FULL = 3

c_void_p = C.c_void_p
c_int = C.c_int
c_long = C.c_long
c_float = C.c_float
c_size_t = C.c_size_t


class LbEncoderLayerWeights(C.Structure):
    _fields_ = [(n, c_void_p) for n in (
        "wqkv_hi", "wqkv_lo", "wkv_hi", "wkv_lo", "wm_hi", "wm_lo", "w1_hi", "w1_lo", "w2_hi", "w2_lo",
        "ln1_g", "ln1_b", "ln2_g", "ln2_b")] + [(n, c_float) for n in ("s_qkv", "s_m", "s_1", "s_2")]


class LbConvWeights(C.Structure):
    _fields_ = [("w_hi", c_void_p), ("w_lo", c_void_p), ("wr_hi", c_void_p), ("wr_lo", c_void_p),
                ("scale", c_void_p), ("shift", c_void_p),
                ("cin", c_int), ("cout", c_int), ("ksize", c_int), ("stride", c_int)]


class LbBackboneWeights(C.Structure):
    _fields_ = [("stem_wt", c_void_p), ("stem_scale", c_void_p), ("stem_shift", c_void_p), ("stem_cout", c_int),
                ("l1", LbConvWeights * 4), ("l2", LbConvWeights * 4), ("l2_down", LbConvWeights),
                ("l3", LbConvWeights * 4), ("l3_down", LbConvWeights), ("l3_out", LbConvWeights),
                ("l2_out", LbConvWeights), ("l2_out2", LbConvWeights * 2), ("l1_out", LbConvWeights),
                ("l1_out2", LbConvWeights * 2)]


class LbTransformerState(C.Structure):
    _fields_ = [("x_f32", c_void_p), ("cat_hi", c_void_p), ("cat_lo", c_void_p), ("mask", c_void_p),
                ("n_groups", c_int), ("group_rows0", c_int), ("group_rows1", c_int), ("n_groups_live", c_void_p)]


class LbCoarseMatchArgs(C.Structure):
    _fields_ = [
        ("f0_hi", c_void_p), ("f0_lo", c_void_p), ("f1_hi", c_void_p), ("f1_lo", c_void_p),
        ("ld", c_int), ("n_pairs", c_int), ("L", c_int), ("S", c_int), ("C", c_int),
        ("h0c", c_int), ("w0c", c_int), ("h1c", c_int), ("w1c", c_int),
        ("match_type", c_int), ("temperature", c_float), ("thr", c_float), ("border_rm", c_int),
        ("bin_score", c_void_p), ("skh_iters", c_int), ("skh_prefilter", c_int),
        ("mask0", c_void_p), ("mask1", c_void_p),
        ("img_scale", c_float), ("scale0", c_void_p), ("scale1", c_void_p),
        ("capacity", c_long),
        ("b_ids", c_void_p), ("i_ids", c_void_p), ("j_ids", c_void_p),
        ("mconf", c_void_p), ("mkpts0_c", c_void_p), ("mkpts1_c", c_void_p), ("count", c_void_p),
        ("conf_matrix", c_void_p),
    ]


class LbFinePreprocessArgs(C.Structure):
    _fields_ = [
        ("feat_f0", c_void_p), ("feat_f1", c_void_p),
        ("sn0", c_long), ("sc0", c_long), ("sh0", c_long), ("sw0", c_long),
        ("sn1", c_long), ("sc1", c_long), ("sh1", c_long), ("sw1", c_long),
        ("Hf0", c_int), ("Wf0", c_int), ("Hf1", c_int), ("Wf1", c_int),
        ("w0c", c_int), ("w1c", c_int), ("stride", c_int), ("W", c_int), ("Cf", c_int), ("Cc", c_int),
        ("feat_c", c_void_p), ("n_pairs", c_int), ("L", c_int), ("S", c_int), ("M", c_long),
        ("b_ids", c_void_p), ("i_ids", c_void_p), ("j_ids", c_void_p),
        ("down_wt", c_void_p), ("down_b", c_void_p), ("merge_w2t", c_void_p), ("merge_b", c_void_p),
        ("merge_w_hi", c_void_p), ("merge_w_lo", c_void_p), ("merge_acc_scale", c_float),
        ("x_f32", c_void_p), ("cat_hi", c_void_p), ("cat_lo", c_void_p),
        ("M_live", c_void_p),
    ]


class LbFineMatchArgs(C.Structure):
    _fields_ = [
        ("f0", c_void_p), ("f1", c_void_p), ("W", c_int), ("C", c_int), ("M", c_long),
        ("img_scale", c_float), ("scale1", c_void_p), ("b_ids", c_void_p), ("mkpts1_c", c_void_p),
        ("expec_f", c_void_p), ("mkpts1_f", c_void_p),
        ("M_live", c_void_p),
    ]


# name -> (restype, argtypes); the same list is what tests/test_host.py checks against the header.
SIGNATURES = {
    "lb_version": (c_int, []),
    "lb_block_k": (c_int, []),
    "lb_conv_layout": (c_int, [c_int, C.POINTER(c_int), C.POINTER(c_int)]),
    "lb_last_error": (C.c_char_p, []),
    "lb_launch_count": (C.c_longlong, []),
    "lb_timing_enable": (c_int, [c_int]),
    "lb_timing_num_tags": (c_int, []),
    "lb_timing_tag_name": (C.c_char_p, [c_int]),
    "lb_timing_collect": (c_int, [C.POINTER(C.c_double), C.POINTER(C.c_longlong), c_int]),
    "lb_split_planes": (c_int, [c_void_p, c_long, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "lb_gemm_split": (c_int, [c_void_p, c_void_p, c_long, c_long, c_void_p, c_void_p, c_long, c_long, c_void_p,
                              c_long, c_long, c_int, c_int, c_int, c_int, c_void_p]),
    "lb_coarse_prep": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                               c_void_p, c_void_p, c_void_p]),
    "lb_backbone_workspace_bytes": (c_size_t, [C.POINTER(LbBackboneWeights), c_int, c_int, c_int]),
    "lb_backbone_forward": (c_int, [C.POINTER(LbBackboneWeights), c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p, c_size_t, c_void_p]),
    "lb_transformer_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "lb_transformer_forward": (c_int, [C.POINTER(LbEncoderLayerWeights), C.POINTER(c_int), c_int, c_int, c_int,
                                       C.POINTER(LbTransformerState), c_void_p, c_size_t, c_void_p]),
    "lb_coarse_match_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "lb_coarse_match": (c_int, [C.POINTER(LbCoarseMatchArgs), c_void_p, c_size_t, c_void_p]),
    "lb_fine_preprocess_workspace_bytes": (c_size_t, [c_long, c_int, c_int]),
    "lb_fine_preprocess": (c_int, [C.POINTER(LbFinePreprocessArgs), c_void_p, c_size_t, c_void_p]),
    "lb_fine_match": (c_int, [C.POINTER(LbFineMatchArgs), c_void_p]),
    "lb_epipolar_errors": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p]),
    "lb_comm_unique_id": (c_int, [C.c_char_p, C.c_char_p]),
    "lb_comm_init": (c_int, [C.c_char_p, c_int, c_int, c_int, C.c_char_p, C.POINTER(c_void_p)]),
    "lb_comm_destroy": (c_int, [c_void_p]),
    "lb_pack_matches": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_long, c_int, c_void_p, c_long, c_void_p]),
    "lb_allgather_matches": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_void_p]),
    "lb_unpack_matches": (c_int, [c_void_p, c_int, c_long, c_void_p, c_void_p, c_void_p, c_void_p, c_long, c_void_p,
                                  c_void_p]),
}

NCCL_UNIQUE_ID_BYTES = 128
# oldest library whose ABI matches the structures above (101: the device-count fields at the end of
# LbTransformerState / LbFinePreprocessArgs / LbFineMatchArgs)
MIN_VERSION = 101
# oldest library that runs full (softmax) attention layers (LAYER_SELF_FULL / LAYER_CROSS_FULL); older ones reject them
FULL_ATTENTION_VERSION = 102


class LibraryMissing(RuntimeError):
    pass


_lib = None


def load():
    """Load libloftr_b200.so (once).  Raises LibraryMissing when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            f"{LIB_PATH} not found: build it with `make` (or `python -c 'import __graft_entry__ as g; g.build()'`). "
            "loftr_b200 has no CPU or PyTorch fallback for the matching hot path.")
    lib = C.CDLL(LIB_PATH)
    lib.lb_version.restype = c_int
    if lib.lb_version() < MIN_VERSION:
        raise LibraryMissing(f"{LIB_PATH} is version {lib.lb_version()}, older than the binding ({MIN_VERSION}): "
                             "rebuild it with `make`")
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def require_full_attention(lib):
    """Raise unless `lib` runs full-attention layers (library version >= FULL_ATTENTION_VERSION)."""
    v = lib.lb_version()
    if v < FULL_ATTENTION_VERSION:
        raise RuntimeError(f"loftr_b200: full attention needs library version {FULL_ATTENTION_VERSION} or newer, but "
                           f"{LIB_PATH} is version {v}: rebuild it with `make`")


def check(rc: int):
    if rc != 0:
        msg = load().lb_last_error()
        raise RuntimeError("loftr_b200: " + (msg.decode() if msg else f"error code {rc}"))


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def timing_enable(on: bool):
    check(load().lb_timing_enable(1 if on else 0))


def timing_collect() -> dict:
    """-> {tag: (total_ms, launches)} for every tensor-core kernel tag recorded since timing_enable(True)."""
    lib = load()
    n = lib.lb_timing_num_tags()
    ms = (C.c_double * n)()
    cnt = (C.c_longlong * n)()
    check(lib.lb_timing_collect(ms, cnt, n))
    return {lib.lb_timing_tag_name(i).decode(): (ms[i], cnt[i]) for i in range(n)}
