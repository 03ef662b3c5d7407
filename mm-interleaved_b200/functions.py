"""Mirror of the reference's ``ops/functions/ms_deform_attn_func.py:24-44``.

``MSDeformAttnFunction.apply(value, shapes, level_start_index, sampling_locations,
attention_weights, im2col_step)`` keeps the reference signature; the forward runs the
sm_90a kernel.  Unlike the reference (``@custom_fwd`` without ``cast_inputs``,
func.py:26), a dtype mismatch between ``value`` and the location / weight tensors --
which the reference op would mis-read (SURVEY.md section 7 hard part iv) -- is resolved by
casting them to ``value.dtype``.
"""
from __future__ import annotations

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import msda as _msda


class MSDeformAttnFunction(Function):
    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations,
                attention_weights, im2col_step):
        ctx.im2col_step = im2col_step
        if sampling_locations.dtype != value.dtype:
            sampling_locations = sampling_locations.to(value.dtype)
        if attention_weights.dtype != value.dtype:
            attention_weights = attention_weights.to(value.dtype)
        output = _msda.ms_deform_attn_forward(
            value.contiguous(), value_spatial_shapes.contiguous(), value_level_start_index.contiguous(),
            sampling_locations.contiguous(), attention_weights.contiguous(), ctx.im2col_step)
        if any(t.requires_grad for t in (value, sampling_locations, attention_weights)):
            ctx.save_for_backward(value, value_spatial_shapes, value_level_start_index,
                                  sampling_locations, attention_weights)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, shapes, starts, loc, attn = ctx.saved_tensors
        grad_value, grad_loc, grad_attn = _msda.ms_deform_attn_backward(
            value, shapes, starts, loc, attn, grad_output.contiguous(), ctx.im2col_step)
        return grad_value, None, None, grad_loc, grad_attn, None
