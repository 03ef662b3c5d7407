"""Autograd Functions over the decoder-layer kernels: the training path of the Llama decoder's self-attention layer.

Each forward runs the same sm_90a kernel as the inference wrapper in ops.py (a Function's forward runs with grad
disabled, so the wrappers' ``inference_only`` guard does not fire there) and saves what its backward kernel reads:

* ``RMSNormFunction``   -- ``mmfs_rmsnorm`` / ``mmfs_rmsnorm_backward`` (dweight only when the weight needs a gradient);
* ``RoPEQKVFunction``   -- ``mmfs_rope_qk`` out of place on the (B, T, 3, H, hd) QKV projection output; the backward
  is the same kernel with the sin table negated (the transpose of a rotation by theta is the rotation by -theta);
* ``AttentionFunction`` -- causal ``mmfs_attn_forward_lse`` on that QKV buffer, saving O and the row log-sum-exp;
  ``mmfs_attn_backward`` writes dQ / dK / dV into one (B, T, 3, H, hd) gradient, so the QKV projection's backward
  stays one GEMM;
* ``SwiGLUFunction``    -- ``mmfs_swiglu`` / ``mmfs_swiglu_backward`` on the [gate | up] buffer.

The backward kernels take bf16 / fp16 only, and the attention backward head dim 128 without a KV cache; other inputs
are refused with the library's message.  Double backward is not supported.
"""
from __future__ import annotations

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ops


class RMSNormFunction(Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        x = x.contiguous()
        ctx.eps = eps
        ctx.save_for_backward(x, weight)
        return ops.rmsnorm(x, weight, eps)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dx, dw = ops.rmsnorm_backward(x, weight, dy.contiguous(), ctx.eps, weight_grad=ctx.needs_input_grad[1])
        return dx, dw, None


class RoPEQKVFunction(Function):
    @staticmethod
    def forward(ctx, qkv, cos, sin, position_ids):
        """``qkv`` (B, T, 3, H, hd); returns a new (B, T, 3, H, hd) tensor with q and k rotated and v copied."""
        out = qkv.contiguous().clone()
        ops.rope_qk_(out[:, :, 0], out[:, :, 1], cos, sin, position_ids)
        ctx.save_for_backward(cos, sin, position_ids)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        cos, sin, position_ids = ctx.saved_tensors
        g = grad.contiguous().clone()
        ops.rope_qk_(g[:, :, 0], g[:, :, 1], cos, torch.neg(sin), position_ids)
        return g, None, None, None


class AttentionFunction(Function):
    @staticmethod
    def forward(ctx, qkv, key_mask, scale):
        """Causal attention over the (B, T, 3, H, hd) ``qkv``; ``key_mask`` (B, T) (1 = attend) or None.  Returns
        (B, T, H * hd)."""
        B, T, _, H, hd = qkv.shape
        out, lse = ops.attention_forward_lse(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], key_mask=key_mask, scale=scale)
        ctx.scale = scale
        ctx.save_for_backward(qkv, out, lse, key_mask)
        return out.view(B, T, H * hd)

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        qkv, out, lse, key_mask = ctx.saved_tensors
        d_out = d_out.contiguous().view(out.shape)
        d_qkv = torch.empty_like(qkv, memory_format=torch.contiguous_format)
        ops.attention_backward(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], out, d_out, lse, d_qkv[:, :, 0], d_qkv[:, :, 1],
                               d_qkv[:, :, 2], key_mask=key_mask, scale=ctx.scale)
        return d_qkv, None, None


class SwiGLUFunction(Function):
    @staticmethod
    def forward(ctx, gate_up):
        gate_up = gate_up.contiguous()
        ctx.save_for_backward(gate_up)
        return ops.swiglu(gate_up)

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        (gate_up,) = ctx.saved_tensors
        return ops.swiglu_backward(gate_up, d_out.contiguous())


def rmsnorm(x, weight, eps):
    return RMSNormFunction.apply(x, weight, eps)


def rope_qkv(qkv, cos, sin, position_ids):
    return RoPEQKVFunction.apply(qkv, cos, sin, position_ids)


def attention(qkv, key_mask=None, scale=None):
    return AttentionFunction.apply(qkv, key_mask, float(scale if scale is not None else qkv.shape[-1] ** -0.5))


def swiglu(gate_up):
    return SwiGLUFunction.apply(gate_up)
