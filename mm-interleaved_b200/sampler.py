"""Tensor-level wrappers of the fused MMFS sampler (csrc/mmfs_sampler_sm100.cu)."""
from __future__ import annotations

import torch

from . import _lib
from .msda import _DTYPE_CODE, _require


def _common(shapes, starts, qproj, rtable, relpos, refpts, scale_ratios, M, n_lvl, P):
    for t, name in ((shapes, "spatial_shapes"), (starts, "level_start_index"), (qproj, "qproj"), (rtable, "rtable"),
                    (relpos, "relpos"), (refpts, "reference_points"), (scale_ratios, "scale_ratios")):
        _require(t.is_cuda and t.is_contiguous(), f"{name} must be a contiguous CUDA tensor")
    _require(qproj.dtype in (torch.float32, torch.float16, torch.bfloat16) and rtable.dtype == qproj.dtype,
             "qproj / rtable must share a float dtype")
    _require(relpos.dtype == torch.uint8 and refpts.dtype == torch.float32 and scale_ratios.dtype == torch.float32,
             "relpos must be uint8, reference_points / scale_ratios fp32")
    _require(shapes.dtype == torch.int64 and starts.dtype == torch.int64, "shape tables must be int64")
    N, Lq, C = qproj.shape
    n_img = relpos.shape[1]
    _require(C == M * P * 2 + M * n_lvl * (P + 1) and rtable.shape[1] == C, "qproj / rtable column count mismatch")
    _require(relpos.shape[0] == N and relpos.shape[2] in (1, Lq), "relpos must be (N, n_img, 1|Lq)")
    _require(shapes.shape[0] == n_img * n_lvl, "spatial_shapes must have n_img * n_levels rows")
    _require(refpts.dim() == 4 and refpts.shape[1] == Lq and refpts.shape[3] == 2, "reference_points must be (1|N, Lq, 1|L, 2)")
    _require(scale_ratios.numel() == n_lvl, "scale_ratios must have n_levels entries")
    return N, Lq, n_img


def mmfs_sampler_forward(value, shapes, starts, qproj, rtable, relpos, refpts, scale_ratios,
                         n_levels: int, n_points: int, want_null_mass: bool = False, strict: bool = False,
                         exact_weights: bool = False, generic: bool = False):
    """Fused relpos lookup + mask + null-slot softmax + location arithmetic + deformable gather.
    Returns the sampled features (N, Lq, M*D) [and the null mass (N, Lq, M) fp32].

    16-bit tensors with D = 64, P = 8 and 3 or 4 levels run the specialised kernel (csrc/mmfs_sampler_v2_sm100.cu),
    whose tap weights are rounded to the element type by default; ``exact_weights`` keeps them fp32 there,
    ``generic`` forces the generic kernel (fp32 tap weights)."""
    from .ops import inference_only
    inference_only("mmfs_sampler_forward", value, qproj, rtable)
    _require(value.is_cuda and value.is_contiguous() and value.dim() == 4, "value must be contiguous CUDA (N,S,M,D)")
    _, S, M, D = value.shape
    N, Lq, n_img = _common(shapes, starts, qproj, rtable, relpos, refpts, scale_ratios, M, n_levels, n_points)
    _require(value.shape[0] == N and value.dtype == qproj.dtype, "value batch / dtype mismatch")
    out = torch.empty((N, Lq, M * D), dtype=value.dtype, device=value.device)
    null_mass = torch.empty((N, Lq, M), dtype=torch.float32, device=value.device) if want_null_mass else None
    if N == 0 or Lq == 0:
        return (out, null_mass) if want_null_mass else out
    with torch.cuda.device(value.device):
        rc = _lib.lib().mmfs_sampler_forward(
            value.data_ptr(), shapes.data_ptr(), starts.data_ptr(), qproj.data_ptr(), rtable.data_ptr(),
            relpos.data_ptr(), refpts.data_ptr(), scale_ratios.data_ptr(), out.data_ptr(),
            null_mass.data_ptr() if want_null_mass else None,
            N, S, M, D, n_img, n_levels, Lq, n_points, relpos.shape[2], refpts.shape[0], refpts.shape[2],
            rtable.shape[0], _DTYPE_CODE[value.dtype],
            (_lib.MSDA_STRICT if strict else 0) |
            (_lib.SAMPLER_EXACT_WEIGHTS if exact_weights else 0) | (_lib.SAMPLER_GENERIC if generic else 0),
            torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "mmfs_sampler_forward")
    return (out, null_mass) if want_null_mass else out


def mmfs_sampler_locw(shapes, starts, qproj, rtable, relpos, refpts, scale_ratios, n_heads: int, n_levels: int,
                      n_points: int):
    """Materialise sampling_locations (N,Lq,M,L,P,2), attention_weights (N,Lq,M,L,P) and the null mass
    exactly as the fused kernel derives them (parity instrumentation / generic-head-size route)."""
    N, Lq, n_img = _common(shapes, starts, qproj, rtable, relpos, refpts, scale_ratios, n_heads, n_levels, n_points)
    L = n_img * n_levels
    loc = torch.empty((N, Lq, n_heads, L, n_points, 2), dtype=qproj.dtype, device=qproj.device)
    attn = torch.empty((N, Lq, n_heads, L, n_points), dtype=qproj.dtype, device=qproj.device)
    null_mass = torch.empty((N, Lq, n_heads), dtype=torch.float32, device=qproj.device)
    if N == 0 or Lq == 0:
        return loc, attn, null_mass
    with torch.cuda.device(qproj.device):
        rc = _lib.lib().mmfs_sampler_locw(
            shapes.data_ptr(), starts.data_ptr(), qproj.data_ptr(), rtable.data_ptr(), relpos.data_ptr(),
            refpts.data_ptr(), scale_ratios.data_ptr(), loc.data_ptr(), attn.data_ptr(), null_mass.data_ptr(),
            N, n_heads, n_img, n_levels, Lq, n_points, relpos.shape[2], refpts.shape[0], refpts.shape[2],
            rtable.shape[0], _DTYPE_CODE[qproj.dtype], torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "mmfs_sampler_locw")
    return loc, attn, null_mass
