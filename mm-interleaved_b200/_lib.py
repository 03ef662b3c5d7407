"""ctypes binding of libmmfs_b200.so (the C ABI declared in include/mmfs_b200.h).

There is NO fallback: if the library is missing or fails to load, importing the ops
raises.  ``MMFS_B200_LIB`` may point at an alternative build of the library.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MMFS_B200_LIB", os.path.join(_HERE, "libmmfs_b200.so"))

OK, EINVAL, EUNSUPPORTED, ECUDA = 0, -1, -2, -3
F32, F16, BF16, F64 = 0, 1, 2, 3
MSDA_STRICT = 1
SAMPLER_EXACT_WEIGHTS = 4
SAMPLER_GENERIC = 8
SELECT_GREEDY, SELECT_SAMPLE = 0, 1

_lib = None

_I, _U, _P = ctypes.c_int, ctypes.c_uint, ctypes.c_void_p
_L, _F = ctypes.c_long, ctypes.c_float

# name -> (restype, argtypes); every symbol include/mmfs_b200.h declares
SIGNATURES = {
    "mmfs_abi_version": (_I, []),
    "mmfs_last_error": (ctypes.c_char_p, []),
    "mmfs_msda_forward": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _U, _P]),
    "mmfs_msda_backward": (_I, [_P] * 9 + [_I] * 8 + [_P]),
    "mmfs_msda_backward_deterministic": (_I, [_P] * 11 + [_I] * 8 + [_P]),
    "mmfs_msda_index_stream": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "mmfs_msda_forward_host": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _U, _P]),
    "mmfs_release_scratch": (None, []),
    "mmfs_sampler_forward": (_I, [_P] * 10 + [_I] * 13 + [_U, _P]),
    "mmfs_sampler_locw": (_I, [_P] * 10 + [_I] * 11 + [_P]),
    "mmfs_rmsnorm": (_I, [_P, _P, _P, _L, _I, _F, _I, _P]),
    "mmfs_layernorm": (_I, [_P, _P, _P, _P, _L, _I, _F, _I, _P]),
    "mmfs_rope_qk": (_I, [_P, _P, _P, _P, _P, _L, _I, _I, _I, _I, _I, _I, _I, _P]),
    "mmfs_rope_qk_append": (_I, [_P] * 9 + [_L, _L] + [_I] * 6 + [_L, _L, _I, _I, _P]),
    "mmfs_swiglu": (_I, [_P, _P, _L, _I, _I, _P]),
    "mmfs_geglu": (_I, [_P, _P, _L, _I, _I, _P]),
    "mmfs_attn_generic": (_I, [_P] * 5 + [_I] * 5 + [_L] * 8 + [_F, _I, _I, _I, _P]),
    "mmfs_groupnorm_nhwc": (_I, [_P] * 5 + [_I] * 4 + [_F, _I, _I, _P]),
    "mmfs_groupnorm_nhwc_backward": (_I, [_P] * 6 + [_I] * 4 + [_F, _I, _I, _P]),
    "mmfs_conv2d_nhwc": (_I, [_P] * 6 + [_I] * 10 + [_P]),
    "mmfs_conv2d_up2x_nhwc": (_I, [_P] * 4 + [_I] * 6 + [_P]),
    "mmfs_conv2d_down2x_nhwc": (_I, [_P] * 4 + [_I] * 6 + [_P]),
    "mmfs_attn_decode_scratch_floats": (_L, [_I] * 4),
    "mmfs_attn_decode": (_I, [_P] * 6 + [_I] * 4 + [_L] * 6 + [_F, _I, _I, _I, _P]),
    "mmfs_attn_decode_shared": (_I, [_P] * 9 + [_I] * 7 + [_L] * 10 + [_F, _I, _I, _I, _P]),
    "mmfs_attn_forward": (_I, [_P] * 5 + [_I] * 5 + [_L] * 8 + [_F, _I, _I, _I, _P, _P]),
    "mmfs_attn_prefix_shared": (_I, [_P] * 8 + [_I] * 6 + [_L] * 12 + [_F, _I, _P, _P]),
    "mmfs_attn_forward_lse": (_I, [_P] * 6 + [_I] * 5 + [_L] * 8 + [_F, _I, _I, _I, _P, _P]),
    "mmfs_attn_backward": (_I, [_P] * 11 + [_I] * 4 + [_L] * 16 + [_F, _I, _P]),
    "mmfs_attn_backward_general": (_I, [_P] * 11 + [_I] * 5 + [_L] * 16 + [_F, _I, _I, _P]),
    "mmfs_rmsnorm_backward": (_I, [_P] * 6 + [_L, _I, _F, _I, _P]),
    "mmfs_layernorm_backward": (_I, [_P] * 7 + [_L, _I, _F, _I, _P]),
    "mmfs_swiglu_backward": (_I, [_P] * 3 + [_L, _I, _I, _P]),
    "mmfs_geglu_backward": (_I, [_P] * 3 + [_L, _I, _I, _P]),
    "mmfs_quick_gelu_backward": (_I, [_P] * 3 + [_L, _I, _P]),
    "mmfs_resize_bilinear_backward": (_I, [_P] * 2 + [_I] * 6 + [_L] * 3 + [_F, _F, _I, _P]),
    "mmfs_decode_select": (_I, [_P, _L] + [_P] * 5 + [_I, _L, _I] + [_P] * 3 + [_I] * 4 + [_P]),
    "mmfs_beam_select": (_I, [_P, _L] + [_P] * 11 + [_I, _L, _I, _P] + [_I] * 4 + [_P]),
    "mmfs_beam_sample": (_I, [_P, _L] + [_P] * 14 + [_I, _L, _I, _I, _P] + [_I] * 4 + [_P]),
    "mmfs_kv_beam_reorder": (_I, [_P, _I, _L, _I, _L, _L, _L, _I] + [_P] * 4 + [_I, _P]),
    "mmfs_image_reentry": (_I, [_P, _P] + [_I] * 5 + [_P]),
    "mmfs_linear_fp8": (_I, [_P] * 6 + [_I] * 4 + [_P]),
    "mmfs_rope_qk_append_fp8": (_I, [_P] * 11 + [_L, _L] + [_I] * 6 + [_L] * 4 + [_I, _I, _P]),
    "mmfs_attn_decode_fp8": (_I, [_P] * 8 + [_I] * 4 + [_L] * 6 + [_F, _I, _I, _I, _P]),
    "mmfs_attn_decode_shared_fp8": (_I, [_P] * 13 + [_I] * 7 + [_L] * 10 + [_F, _I, _I, _I, _P]),
    "mmfs_kv_dequantize_fp8": (_I, [_P] * 3 + [_I] * 4 + [_L] * 6 + [_I, _P]),
}
BEAM_MAX_BEAMS, BEAM_MAX_EOS = 8, 4                  # limits of mmfs_beam_select / mmfs_beam_sample / mmfs_kv_beam_reorder
LINEAR_FP8_MAX_M = 64                                # rows of x mmfs_linear_fp8 takes
RMSNORM_BWD_PARTS = 256                              # MMFS_RMSNORM_BWD_PARTS: dweight partial rows of mmfs_rmsnorm_backward


def lib() -> ctypes.CDLL:
    """Load (once) and return the library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"libmmfs_b200.so not found at {LIB_PATH}: build it with "
                "`python mm-interleaved_b200/build.py` (there is no CPU / PyTorch fallback)")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the ABI is incomplete
            fn.restype = res
            fn.argtypes = args
        if handle.mmfs_abi_version() != 3:
            raise RuntimeError(f"libmmfs_b200.so ABI {handle.mmfs_abi_version()} != 3")
        _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    """Turn a negative status into the RuntimeError the reference extension would raise."""
    if rc != OK:
        msg = lib().mmfs_last_error().decode("utf-8", "replace")
        kind = {EINVAL: "invalid argument", EUNSUPPORTED: "unsupported", ECUDA: "CUDA error"}.get(rc, "error")
        raise RuntimeError(f"{what}: {kind} ({rc}): {msg}")
