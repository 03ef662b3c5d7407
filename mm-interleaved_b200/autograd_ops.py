"""Autograd Functions over the decoder-layer kernels: the training path of the Llama decoder's self-attention layer
and of the visual tokenizer's Q-Former head.

Each forward runs the same sm_90a kernel as the inference wrapper in ops.py (a Function's forward runs with grad
disabled, so the wrappers' ``inference_only`` guard does not fire there) and saves what its backward kernel reads:

* ``RMSNormFunction``   -- ``mmfs_rmsnorm`` / ``mmfs_rmsnorm_backward`` (dweight only when the weight needs a gradient);
* ``RoPEQKVFunction``   -- ``mmfs_rope_qk`` out of place on the (B, T, 3, H, hd) QKV projection output; the backward
  is the same kernel with the sin table negated (the transpose of a rotation by theta is the rotation by -theta);
* ``AttentionFunction`` -- causal ``mmfs_attn_forward_lse`` on that QKV buffer, saving O and the row log-sum-exp;
  ``mmfs_attn_backward`` writes dQ / dK / dV into one (B, T, 3, H, hd) gradient, so the QKV projection's backward
  stays one GEMM; non-causal (CLIP's patch self-attention) on ``mmfs_attn_backward_general`` into the same buffer;
* ``SwiGLUFunction``    -- ``mmfs_swiglu`` / ``mmfs_swiglu_backward`` on the [gate | up] buffer;
* ``LayerNormFunction`` -- ``mmfs_layernorm`` / ``mmfs_layernorm_backward`` (dweight / dbias only when asked for);
* ``GeneralAttentionFunction`` -- non-causal ``mmfs_attn_forward_lse`` on separate q (B, Tq, H, hd) and k / v
  (B, Tkv, H, hd) with an optional (B, Tkv) key mask (the Q-Former's self- and cross-attention);
  ``mmfs_attn_backward_general`` returns dq, dk, dv;
* ``QuickGELUFunction`` -- CLIP's ``h * sigmoid(1.702 h)`` in torch ops (the inference path's bits), backward on
  ``mmfs_quick_gelu_backward``; saves h only;
* ``ResizeBilinearFunction`` -- ``F.interpolate(scale_factor=s, mode="bilinear")`` forward (the inference path's
  bits), backward on ``mmfs_resize_bilinear_backward`` straight into the token layout of the input.

The backward kernels take bf16 / fp16 only, the causal attention backward head dim 128 without a KV cache and the
general one head dim 64 or 128; other inputs are refused with the library's message.  Double backward is not
supported.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
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
    def forward(ctx, qkv, key_mask, scale, causal):
        """Causal (or not) attention over the (B, T, 3, H, hd) ``qkv``; ``key_mask`` (B, T) (1 = attend) or None.
        Returns (B, T, H * hd)."""
        B, T, _, H, hd = qkv.shape
        out, lse = ops.attention_forward_lse(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], key_mask=key_mask, scale=scale,
                                             causal=causal)
        ctx.scale, ctx.causal = scale, causal
        ctx.save_for_backward(qkv, out, lse, key_mask)
        return out.view(B, T, H * hd)

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        qkv, out, lse, key_mask = ctx.saved_tensors
        d_out = d_out.contiguous().view(out.shape)
        d_qkv = torch.empty_like(qkv, memory_format=torch.contiguous_format)
        bwd = ops.attention_backward if ctx.causal else ops.attention_backward_general
        bwd(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], out, d_out, lse, d_qkv[:, :, 0], d_qkv[:, :, 1], d_qkv[:, :, 2],
            key_mask=key_mask, scale=ctx.scale)
        return d_qkv, None, None, None


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


class LayerNormFunction(Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        x = x.contiguous()
        ctx.eps = eps
        ctx.save_for_backward(x, weight)
        return ops.layernorm(x, weight, bias, eps)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dx, dw, db = ops.layernorm_backward(x, weight, dy.contiguous(), ctx.eps, weight_grad=ctx.needs_input_grad[1],
                                            bias_grad=ctx.needs_input_grad[2])
        return dx, dw, db, None


class GeneralAttentionFunction(Function):
    @staticmethod
    def forward(ctx, q, k, v, key_mask, scale):
        """Non-causal attention of q (B, Tq, H, hd) over k / v (B, Tkv, H, hd) (dense heads, any batch / token strides);
        ``key_mask`` (B, Tkv) (1 = attend) or None.  Returns (B, Tq, H * hd)."""
        B, Tq, H, hd = q.shape
        out, lse = ops.attention_forward_lse(q, k, v, key_mask=key_mask, scale=scale, causal=False)
        ctx.scale = scale
        ctx.save_for_backward(q, k, v, out, lse, key_mask)
        return out.view(B, Tq, H * hd)

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        q, k, v, out, lse, key_mask = ctx.saved_tensors
        d_out = d_out.contiguous().view(out.shape)
        dq = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        dk = torch.empty(k.shape, dtype=k.dtype, device=k.device)
        dv = torch.empty(v.shape, dtype=v.dtype, device=v.device)
        ops.attention_backward_general(q, k, v, out, d_out, lse, dq, dk, dv, key_mask=key_mask, scale=ctx.scale)
        return dq, dk, dv, None, None


class QuickGELUFunction(Function):
    @staticmethod
    def forward(ctx, h):
        ctx.save_for_backward(h)
        return h * torch.sigmoid(1.702 * h)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        (h,) = ctx.saved_tensors
        return ops.quick_gelu_backward(h.contiguous(), dy.contiguous())


class ResizeBilinearFunction(Function):
    @staticmethod
    def forward(ctx, x, scale_factor):
        """``x`` (B, C, H, W), any strides; returns F.interpolate(x, scale_factor, bilinear, align_corners=False)."""
        ctx.scale_factor, ctx.in_hw = scale_factor, x.shape[2:]
        return F.interpolate(x, scale_factor=scale_factor, mode="bilinear", align_corners=False)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        B, C = dy.shape[:2]
        H, W = ctx.in_hw
        dx = ops.resize_bilinear_backward(dy, (H, W), ctx.scale_factor)           # (B, H * W, C)
        return dx.view(B, H, W, C).permute(0, 3, 1, 2), None


def rmsnorm(x, weight, eps):
    return RMSNormFunction.apply(x, weight, eps)


def rope_qkv(qkv, cos, sin, position_ids):
    return RoPEQKVFunction.apply(qkv, cos, sin, position_ids)


def attention(qkv, key_mask=None, scale=None, causal=True):
    return AttentionFunction.apply(qkv, key_mask, float(scale if scale is not None else qkv.shape[-1] ** -0.5), causal)


def swiglu(gate_up):
    return SwiGLUFunction.apply(gate_up)


def layernorm(x, weight, bias, eps):
    return LayerNormFunction.apply(x, weight, bias, eps)


def attention_general(q, k, v, key_mask=None, scale=None):
    return GeneralAttentionFunction.apply(q, k, v, key_mask, float(scale if scale is not None else q.shape[-1] ** -0.5))


def quick_gelu(h):
    return QuickGELUFunction.apply(h)


def resize_bilinear(x, scale_factor):
    return ResizeBilinearFunction.apply(x, scale_factor)
