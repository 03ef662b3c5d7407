"""Tensor-level entry points of the native op, mirroring the reference extension module
``MultiScaleDeformableAttention`` (ops/src/vision.cpp:13-16, ops/src/ms_deform_attn.h:20-61).

Host code stays PyTorch (device memory, streams); the arithmetic is the hand-written
sm_90a kernel behind the C ABI (csrc/msda_fwd_sm100.cu).
"""
from __future__ import annotations

import torch

from . import _lib

_DTYPE_CODE = {torch.float32: _lib.F32, torch.float16: _lib.F16, torch.bfloat16: _lib.BF16,
               torch.float64: _lib.F64}


def _require(cond: bool, msg: str) -> None:
    if not cond:
        raise RuntimeError(msg)


def _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
    # preconditions of ms_deform_attn_cuda_forward, cu:29-53, same messages
    _require(value.is_contiguous(), "value tensor has to be contiguous")
    _require(spatial_shapes.is_contiguous(), "spatial_shapes tensor has to be contiguous")
    _require(level_start_index.is_contiguous(), "level_start_index tensor has to be contiguous")
    _require(sampling_loc.is_contiguous(), "sampling_loc tensor has to be contiguous")
    _require(attn_weight.is_contiguous(), "attn_weight tensor has to be contiguous")
    if not value.is_cuda:
        raise RuntimeError("Not implemented on the CPU")          # ms_deform_attn.h:38
    _require(spatial_shapes.is_cuda, "spatial_shapes must be a CUDA tensor")
    _require(level_start_index.is_cuda, "level_start_index must be a CUDA tensor")
    _require(sampling_loc.is_cuda, "sampling_loc must be a CUDA tensor")
    _require(attn_weight.is_cuda, "attn_weight must be a CUDA tensor")
    _require(value.dim() == 4 and sampling_loc.dim() == 6 and attn_weight.dim() == 5,
             "expected value (N,S,M,D), sampling_loc (N,Lq,M,L,P,2), attn_weight (N,Lq,M,L,P)")
    _require(value.dtype in _DTYPE_CODE, f"unsupported dtype {value.dtype}")
    # the reference reads shapes through data<int64_t>() and the float tensors through
    # data<scalar_t>() of value's type (cu:67-72): a mismatch is an error there too
    _require(spatial_shapes.dtype == torch.int64 and level_start_index.dtype == torch.int64,
             "spatial_shapes / level_start_index must be int64")
    _require(sampling_loc.dtype == value.dtype and attn_weight.dtype == value.dtype,
             "sampling_loc / attn_weight must have value's dtype")
    N, S, M, D = value.shape
    L = spatial_shapes.shape[0]
    Lq, P = sampling_loc.shape[1], sampling_loc.shape[4]
    _require(tuple(spatial_shapes.shape) == (L, 2) and level_start_index.numel() == L,
             "spatial_shapes must be (L,2) and level_start_index (L,)")
    _require(tuple(sampling_loc.shape) == (N, Lq, M, L, P, 2), "sampling_loc shape mismatch")
    _require(tuple(attn_weight.shape) == (N, Lq, M, L, P), "attn_weight shape mismatch")
    step = min(N, int(im2col_step)) if N > 0 else 1
    _require(step > 0 and N % step == 0,
             f"batch({N}) must divide im2col_step({step})")        # cu:51-53
    return N, S, M, D, L, Lq, P


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                           im2col_step: int = 64, strict: bool = False, w16: bool = False) -> torch.Tensor:
    """Drop-in for ``MSDA.ms_deform_attn_forward`` (ops/src/ms_deform_attn.h:20-39).

    Returns a new tensor (N, Lq, M*D) with value's dtype/device (cu:55,78).  All N samples go
    through one launch on the current stream; ``im2col_step`` is validated like the
    reference does but does not change the result.  bf16 is accepted (superset).
    """
    N, S, M, D, L, Lq, P = _check_inputs(value, spatial_shapes, level_start_index, sampling_loc,
                                         attn_weight, im2col_step)
    out = torch.empty((N, Lq, M * D), dtype=value.dtype, device=value.device)
    if N == 0 or Lq == 0:
        return out
    with torch.cuda.device(value.device):
        stream = torch.cuda.current_stream().cuda_stream
        rc = _lib.lib().mmfs_msda_forward(
            value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(),
            sampling_loc.data_ptr(), attn_weight.data_ptr(), out.data_ptr(),
            N, S, M, D, L, Lq, P, _DTYPE_CODE[value.dtype],
            (_lib.MSDA_STRICT if strict else 0) | (_lib.MSDA_W16 if w16 else 0), stream)
    _lib.check(rc, "ms_deform_attn_forward")
    return out


def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                            grad_output, im2col_step: int = 64, deterministic: bool = True):
    """Drop-in for ``MSDA.ms_deform_attn_backward`` (ops/src/ms_deform_attn.h:41-61): returns
    ``[grad_value, grad_sampling_loc, grad_attn_weight]`` shaped and typed like the inputs.  Gradients are accumulated
    in fp32 and cast back for 16-bit inputs exactly like the reference host code (cu:122-129, 156-160).  fp64 inputs
    are not implemented (the reference uses them only as ground truth in its test scripts).

    ``deterministic`` (default): ``grad_value`` is reduced with integer atomics on a 64-bit fixed-point buffer, so
    repeated runs are bit-identical (SURVEY.md 8 f4); ``False`` takes the reference's float-atomic scheme (faster,
    last bits vary with the arrival order of the taps)."""
    N, S, M, D, L, Lq, P = _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step)
    _require(grad_output.is_cuda and grad_output.is_contiguous() and grad_output.dtype == value.dtype and
             tuple(grad_output.shape) == (N, Lq, M * D), "grad_output must be a contiguous CUDA tensor (N, Lq, M*D) of value's dtype")
    if value.dtype == torch.float64:
        raise NotImplementedError("ms_deform_attn_backward: float64 is not implemented on the H100 path")
    gl = torch.empty((N, Lq, M, L, P, 2), dtype=torch.float32, device=value.device)
    ga = torch.empty((N, Lq, M, L, P), dtype=torch.float32, device=value.device)
    if deterministic:
        # grad_value accumulated as 64-bit fixed point with integer atomics: bit-reproducible from run to run
        gv = torch.empty((N, S, M, D), dtype=torch.float32, device=value.device)
        fixed = torch.zeros((N, S, M, D), dtype=torch.int64, device=value.device)
        scratch = torch.empty((2,), dtype=torch.float32, device=value.device)
        if N > 0 and Lq > 0:
            with torch.cuda.device(value.device):
                rc = _lib.lib().mmfs_msda_backward_deterministic(
                    value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(), sampling_loc.data_ptr(),
                    attn_weight.data_ptr(), grad_output.data_ptr(), fixed.data_ptr(), gv.data_ptr(), gl.data_ptr(), ga.data_ptr(),
                    scratch.data_ptr(), N, S, M, D, L, Lq, P, _DTYPE_CODE[value.dtype], torch.cuda.current_stream().cuda_stream)
            _lib.check(rc, "ms_deform_attn_backward (deterministic)")
        else:
            gv.zero_()
    else:
        gv = torch.zeros((N, S, M, D), dtype=torch.float32, device=value.device)
        if N > 0 and Lq > 0:
            with torch.cuda.device(value.device):
                rc = _lib.lib().mmfs_msda_backward(
                    value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(), sampling_loc.data_ptr(),
                    attn_weight.data_ptr(), grad_output.data_ptr(), gv.data_ptr(), gl.data_ptr(), ga.data_ptr(),
                    N, S, M, D, L, Lq, P, _DTYPE_CODE[value.dtype], torch.cuda.current_stream().cuda_stream)
            _lib.check(rc, "ms_deform_attn_backward")
    return [gv.to(value.dtype), gl.to(value.dtype), ga.to(value.dtype)]


def msda_index_stream(spatial_shapes, level_start_index, sampling_loc, M: int, D: int) -> torch.Tensor:
    """int32 (N,Lq,M,L,P,8) index stream of the sampler (parity instrumentation)."""
    _require(sampling_loc.is_cuda and sampling_loc.is_contiguous() and sampling_loc.dim() == 6,
             "sampling_loc must be a contiguous CUDA tensor (N,Lq,M,L,P,2)")
    N, Lq, M_, L, P, _ = sampling_loc.shape
    _require(M_ == M, "head count mismatch")
    idx = torch.empty((N, Lq, M, L, P, 8), dtype=torch.int32, device=sampling_loc.device)
    with torch.cuda.device(sampling_loc.device):
        rc = _lib.lib().mmfs_msda_index_stream(
            spatial_shapes.data_ptr(), level_start_index.data_ptr(), sampling_loc.data_ptr(),
            idx.data_ptr(), N, M, D, L, Lq, P, _DTYPE_CODE[sampling_loc.dtype],
            torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "msda_index_stream")
    return idx


def ms_deform_attn_forward_host(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                                out=None, strict: bool = False) -> torch.Tensor:
    """The op through HOST tensors (ideally pinned): H2D copies, kernel, D2H copy and a stream
    synchronise all happen inside ``mmfs_msda_forward_host``.  This is the end-to-end form
    timed as ``e2e`` by bench.py."""
    for t in (value, spatial_shapes, level_start_index, sampling_loc, attn_weight):
        _require(not t.is_cuda and t.is_contiguous(), "host entry point takes contiguous CPU tensors")
    N, S, M, D = value.shape
    L = spatial_shapes.shape[0]
    Lq, P = sampling_loc.shape[1], sampling_loc.shape[4]
    if out is None:
        out = torch.empty((N, Lq, M * D), dtype=value.dtype, pin_memory=True)
    rc = _lib.lib().mmfs_msda_forward_host(
        value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(),
        sampling_loc.data_ptr(), attn_weight.data_ptr(), out.data_ptr(),
        N, S, M, D, L, Lq, P, _DTYPE_CODE[value.dtype], _lib.MSDA_STRICT if strict else 0,
        torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "ms_deform_attn_forward_host")
    return out
