"""ctypes binding of libfatezero_b200.so (the C ABI declared in include/fatezero_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# FZ_LIB_VARIANT=<suffix> loads libfatezero_b200_<suffix>.so: a development aid for A/B-ing kernel variants built with
# `python fatezero_b200/_build.py --variant <suffix> --flags "-D..."` inside one GPU session (never set by the product path).
_VARIANT = os.environ.get("FZ_LIB_VARIANT", "")
LIB_PATH = os.path.join(_HERE, f"libfatezero_b200_{_VARIANT}.so" if _VARIANT else "libfatezero_b200.so")

c_void_p, c_int, c_ll, c_float = C.c_void_p, C.c_int, C.c_longlong, C.c_float


class Epilogue(C.Structure):
    """fz_epilogue_t"""
    _fields_ = [
        ("bias", c_void_p), ("group_bias", c_void_p), ("rows_per_group", c_int), ("residual", c_void_p), ("ldr", c_ll),
        ("residual2", c_void_p), ("ldr2", c_ll), ("mode", c_int), ("vt_col_start", c_int), ("out_vt", c_void_p), ("vt_S", c_int), ("vt_d", c_int),
        ("vt_heads", c_int), ("vt_ld", c_int),
    ]


class AttnArgs(C.Structure):
    """fz_attn_args_t"""
    _fields_ = [
        ("q", c_void_p), ("ldq", c_ll), ("k", c_void_p), ("ldk", c_ll), ("vt", c_void_p), ("vt_ld", c_ll),
        ("out", c_void_p), ("ldo", c_ll),
        ("S_q", c_int), ("keys_per_slot", c_int), ("n_slots", c_int), ("n_src", c_int),
        ("d", c_int), ("heads", c_int), ("F", c_int), ("BF", c_int),
        ("scale", c_float), ("src_index", C.POINTER(c_int)), ("edit_bf_start", c_int), ("row_mode", c_int),
        ("store", c_void_p), ("base", c_void_p), ("cache_ld", c_ll), ("acc", c_void_p), ("acc_ld", c_ll),
        ("xedit", c_void_p), ("mask", c_void_p), ("dbg", c_void_p), ("causal", c_int),
    ]


MAX_ATTN_GROUPS = 8


class AttnGroup(C.Structure):
    """fz_attn_group_t"""
    _fields_ = [("row_mode", c_int), ("xedit", c_void_p), ("mask", c_void_p), ("acc", c_void_p)]


class AttnGroups(C.Structure):
    """fz_attn_groups_t"""
    _fields_ = [("n_groups", c_int), ("g", AttnGroup * MAX_ATTN_GROUPS)]


class AttnSlabs(C.Structure):
    """fz_attn_slabs_t"""
    _fields_ = [("store", c_void_p * MAX_ATTN_GROUPS), ("base", c_void_p * MAX_ATTN_GROUPS)]


class P2PSeg(C.Structure):
    """fz_p2p_seg_t"""
    _fields_ = [("src", c_void_p), ("src_pitch", c_ll), ("dst", c_void_p), ("dst_pitch", c_ll), ("rows", c_int), ("row_bytes", c_int),
                ("dst_slot", c_int)]


EPI_ROWMAJOR, EPI_GEGLU = 0, 1
ATTN_NONE, ATTN_STORE, ATTN_REPLACE, ATTN_BLEND, ATTN_CROSSEDIT = 0, 1, 2, 3, 4
XEDIT_FLOATS = 8 + 4 * 80 + 80 * 80

# name -> argtypes (every function returns int); MUST list every symbol of include/fatezero_b200.h
SIGNATURES = {
    "fz_gemm_f16": [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, C.POINTER(Epilogue), c_void_p, c_ll, c_int, c_void_p],
    "fz_conv3x3_nhwc_f16": [c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, C.POINTER(Epilogue), c_void_p, c_ll,
                            c_int, c_void_p],
    "fz_conv3x3_down_asym_nhwc_f16": [c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p, c_int, C.POINTER(Epilogue), c_void_p, c_ll, c_int,
                                      c_void_p],
    "fz_tconv3_f16": [c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p, c_int, C.POINTER(Epilogue), c_void_p, c_ll, c_int, c_void_p],
    "fz_tconv3_halo_f16": [c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p, c_int, C.POINTER(Epilogue), c_void_p, c_ll, c_int, c_void_p],
    "fz_attention_f16": [C.POINTER(AttnArgs), c_void_p],
    "fz_attention_grouped_f16": [C.POINTER(AttnArgs), C.POINTER(AttnGroups), c_void_p],
    "fz_attention_grouped_slabs_f16": [C.POINTER(AttnArgs), C.POINTER(AttnGroups), C.POINTER(AttnSlabs), c_void_p],
    "fz_groupnorm_nhwc_f16": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_int, c_void_p,
                              c_void_p],
    "fz_groupnorm_batched_nhwc_f16": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_int,
                                      c_void_p, c_void_p],
    "fz_groupnorm_stats_f16": [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "fz_groupnorm_apply_f16": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_int, c_void_p,
                               c_void_p],
    "fz_groupnorm_apply_sums64_f16": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_int,
                                      c_void_p, c_void_p],
    "fz_layernorm_f16": [c_void_p, c_void_p, c_ll, c_int, c_void_p, c_void_p, c_float, c_void_p],
    "fz_upsample2x_nhwc_f16": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "fz_concat_channels_f16": [c_void_p, c_int, c_void_p, c_int, c_void_p, c_ll, c_void_p],
    "fz_im2col_latents_f16": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "fz_out_temporal_f32": [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                            c_void_p],
    "fz_rowvec_linear": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "fz_timestep_sinusoid": [c_float, c_void_p, c_int, c_int, c_float, c_void_p],
    "fz_temporal_attn_f16": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p],
    "fz_ddim_invert_step": [c_void_p, c_void_p, c_ll, c_float, c_float, c_void_p],
    "fz_cfg_ddim_step": [c_void_p, c_void_p, c_ll, c_float, c_float, c_float, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "fz_cfg_ddim_step_batched": [c_void_p, c_void_p, c_int, c_ll, c_float, c_float, c_float, c_void_p, C.POINTER(c_void_p),
                                 C.POINTER(c_void_p), C.POINTER(c_int), c_ll, c_void_p],
    "fz_cfg_ddim_step_multi": [c_void_p, c_void_p, c_int, c_ll, c_float, c_float, c_float, C.POINTER(c_void_p), C.POINTER(c_void_p),
                               C.POINTER(c_void_p), C.POINTER(c_int), c_ll, c_void_p],
    "fz_blend_mask": [C.POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int, c_int, C.POINTER(c_float), c_float, c_int, c_int,
                      c_void_p, c_void_p],
    "fz_p2p_alloc": [c_ll, C.POINTER(c_void_p)],
    "fz_p2p_free": [c_void_p],
    "fz_p2p_export": [c_void_p, c_void_p],
    "fz_p2p_import": [c_void_p, C.POINTER(c_void_p)],
    "fz_p2p_unimport": [c_void_p],
    "fz_p2p_push": [C.POINTER(P2PSeg), c_int, C.POINTER(c_void_p), c_void_p, c_int, c_void_p, C.c_uint, c_void_p],
    "fz_p2p_wait": [c_void_p, C.c_uint, c_void_p],
    "fz_gn_combine": [c_void_p, C.POINTER(c_void_p), c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "fz_softmax_rows_f16": [c_void_p, c_ll, c_int, c_ll, c_float, c_void_p],
    "fz_embed_tokens_f16": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "fz_quick_gelu_f16": [c_void_p, c_ll, c_void_p],
    "fz_gelu_f16": [c_void_p, c_ll, c_void_p],
    "fz_cross_heatmaps": [C.POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "fz_frames_to_u8": [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p],
    "fz_resize_bicubic_u8": [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                             c_void_p, c_void_p, c_void_p],
    "fz_clip_patchify_f16": [c_void_p, c_int, c_int, c_int, c_int, c_int, C.POINTER(c_float), C.POINTER(c_float), c_void_p, c_void_p],
    "fz_clip_embed_f16": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_void_p, c_void_p],
    "fz_clip_scores": [c_void_p, c_void_p, c_int, c_int, c_int, C.POINTER(c_int), C.POINTER(c_int), c_int, c_float, c_void_p, c_void_p,
                       c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "fz_device_check": [],
    "fz_init": [c_void_p],
    "fz_version": [],
}

_lib = None
launch_count = 0     # C-ABI compute calls issued
kernel_launches = 0  # kernels of this library launched (bench.py reports the delta over its timed region)
KERNELS_PER_CALL = {"fz_groupnorm_nhwc_f16": 2, "fz_groupnorm_batched_nhwc_f16": 2, "fz_p2p_alloc": 0, "fz_p2p_free": 0, "fz_p2p_export": 0, "fz_p2p_import": 0,
                    "fz_p2p_unimport": 0, "fz_init": 0, "fz_resize_bicubic_u8": 2}  # stats + apply (plus one memset); horizontal + vertical
# pass; every other entry point launches one kernel


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(fatezero_b200 has no CPU or PyTorch fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c_int
    lib.fz_last_error.restype = C.c_char_p
    lib.fz_last_error.argtypes = []
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().fz_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


# FZ_ABLATE=<entry point>[,<entry point>...]: timing-only development aid (tools/ablate.py) — the named entry points return without
# launching, so the wall-clock delta of a clip is that kernel class's in-situ cost.  Results are garbage; never set by the product.
_ABLATE = frozenset(x for x in os.environ.get("FZ_ABLATE", "").split(",") if x)


def call(name: str, *args):
    global launch_count, kernel_launches
    lib = load()
    if _ABLATE and name in _ABLATE:
        return
    launch_count += 1
    kernel_launches += KERNELS_PER_CALL.get(name, 1)
    check(getattr(lib, name)(*args), name)
