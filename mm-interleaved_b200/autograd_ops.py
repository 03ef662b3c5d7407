"""The switch between the inference path and the training path, and the autograd Functions of the training path: the
Llama decoder's self-attention layer, the visual tokenizer, and the image loss through the frozen SD UNet.

The entry points at the bottom (``layernorm``, ``rmsnorm``, ``swiglu``, ``geglu``, ``quick_gelu``, ``resize_bilinear``,
``attention``, ``attention_general``, ``group_norm_nhwc``, ``conv``) are the one call a model module makes for the op.
Each decides the path itself: unless autograd records the call (``msda.records``: grad mode on and a tensor argument or
a parameter requires grad) it makes the inference call -- the ops.py kernel, or the torch expression the inference
code computes -- and otherwise it refuses a dtype its backward kernels do not take (``check_training_dtype``, before
any work rather than in ``loss.backward()``) and applies the Function.  ``rope_qkv`` is Function-only: its one caller
is the Llama training forward.

Each Function's forward runs the same sm_90a kernel as the inference wrapper in ops.py (a Function's forward runs with
grad disabled, so the wrappers' ``inference_only`` guard does not fire there) and saves what its backward kernel reads:

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
  bits), backward on ``mmfs_resize_bilinear_backward`` straight into the token layout of the input;
* ``ConvFunction`` -- the SD UNet's convolution with its fused time-embedding add and residual, forward exactly the
  inference ``ops.conv2d`` call; the backward gives dx and d residual with the filter frozen (``conv_input_grad``);
* ``GroupNormNHWCFunction`` -- ``mmfs_groupnorm_nhwc`` (+ SiLU) / ``mmfs_groupnorm_nhwc_backward``, saves x only;
  frozen affine parameters;
* ``GEGLUFunction`` -- ``mmfs_geglu`` / ``mmfs_geglu_backward`` on the [value | gate] buffer.

The backward kernels take bf16 / fp16 only, except the GroupNorm backward and the convolution's data gradient (cuDNN
where the kernels do not apply), which take fp32 too; the causal attention backward takes head dim 128 without a KV
cache and the general one head dim 64 or 128, other head dims are refused with the library's message.  Double
backward is not supported.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ops
from .msda import records


def check_training_dtype(what, t):
    if t.dtype not in (torch.bfloat16, torch.float16):
        raise RuntimeError(f"{what}: the backward kernels take bf16 / fp16 only (got {t.dtype}); cast the model, or run "
                           "under torch.no_grad()")


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


def _refuse_trainable(what, *params):
    """The Functions below give no gradient to these tensors: refuse to drop one silently."""
    if any(p is not None and p.requires_grad for p in params):
        raise RuntimeError(f"{what}: the UNet's own weights have no backward here (the image loss trains what feeds the "
                           "UNet); freeze them, e.g. unet.requires_grad_(False)")


def conv_input_grad(conv, dy: torch.Tensor, x_shape) -> torch.Tensor:
    """dx of ``conv`` (a ``unet_sd.Conv2d``: 3x3 / pad 1 or 1x1 / pad 0 at stride 1, or 3x3 / pad 1 at stride 2) for an
    input of shape ``x_shape`` and output gradient ``dy``.

    * stride 1: dx is the same convolution of dy with the channel-transposed, 180-degree-rotated filter
      (``ops.dgrad_weights_khwc``) on the wgmma kernel;
    * stride 2: dx at the 2H x 2W input is four 2x2 phase convolutions over the H x W dy, the ``conv2d_up2x`` kernel with
      the filter folded by ``ops.fold_dgrad_down2x_weights``;
    * where the swapped channel counts or the tile rule rule the kernels out, ``torch.nn.grad.conv2d_input`` (cuDNN)."""
    w = conv.weight
    stride, pad = conv.stride[0], conv.padding[0]
    K = w.shape[-1]
    if dy.is_cuda and not dy.is_contiguous(memory_format=torch.channels_last):
        dy = dy.contiguous(memory_format=torch.channels_last)
    wt = w.transpose(0, 1)                                      # (Cin, Cout, K, K): the dgrad's channel roles
    if stride == 1 and 2 * pad == K - 1 and ops.conv2d_supported(dy, wt, 1, pad):
        return ops.conv2d(dy, conv.weight_dgrad_khwc(), None, 1, pad)
    if (stride == 2 and K == 3 and pad == 1 and tuple(x_shape[2:]) == (2 * dy.shape[2], 2 * dy.shape[3])
            and ops.conv2d_up2x_supported(dy, wt)):
        return ops.conv2d_up2x(dy, conv.weight_dgrad_down2x())
    return torch.nn.grad.conv2d_input(tuple(x_shape), w, dy, stride=stride, padding=pad)


class ConvFunction(Function):
    @staticmethod
    def forward(ctx, x, residual, conv, add_bc):
        """``conv(x) [+ add_bc[:, :, None, None]] [+ residual]`` as the inference path computes it (``conv.fused``);
        ``conv``'s filter, bias and ``add_bc`` (the time-embedding projection) carry no gradient."""
        _refuse_trainable("ConvFunction", conv.weight, conv.bias, add_bc)
        ctx.conv, ctx.x_shape = conv, tuple(x.shape)
        return conv.fused(x, add_bc, residual)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        dx = conv_input_grad(ctx.conv, dy, ctx.x_shape) if ctx.needs_input_grad[0] else None
        return dx, (dy if ctx.needs_input_grad[1] else None), None, None


class GroupNormNHWCFunction(Function):
    @staticmethod
    def forward(ctx, x, weight, bias, groups, eps, silu):
        _refuse_trainable("GroupNormNHWCFunction", weight, bias)
        ctx.groups, ctx.eps, ctx.silu = groups, eps, silu
        ctx.save_for_backward(x, weight, bias)
        return ops.group_norm_nhwc(x, groups, weight, bias, eps, silu=silu)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight, bias = ctx.saved_tensors
        dx = ops.group_norm_nhwc_backward(x, dy, ctx.groups, weight, bias, ctx.eps, silu=ctx.silu)
        return dx, None, None, None, None, None


class GEGLUFunction(Function):
    @staticmethod
    def forward(ctx, value_gate):
        value_gate = value_gate.contiguous()
        ctx.save_for_backward(value_gate)
        return ops.geglu(value_gate)

    @staticmethod
    @once_differentiable
    def backward(ctx, d_out):
        (value_gate,) = ctx.saved_tensors
        return ops.geglu_backward(value_gate, d_out.contiguous())


def rmsnorm(x, weight, eps):
    if not records(x, weight):
        return ops.rmsnorm(x.contiguous(), weight, eps)
    check_training_dtype("rmsnorm", x)
    return RMSNormFunction.apply(x, weight.to(x.dtype), eps)


def rope_qkv(qkv, cos, sin, position_ids):
    return RoPEQKVFunction.apply(qkv, cos, sin, position_ids)


def attention(qkv, key_mask=None, scale=None, causal=True):
    if not records(qkv):
        return ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], key_mask=key_mask, scale=scale, causal=causal)
    check_training_dtype("attention", qkv)
    return AttentionFunction.apply(qkv, key_mask, float(scale if scale is not None else qkv.shape[-1] ** -0.5), causal)


def swiglu(gate_up):
    if not records(gate_up):
        return ops.swiglu(gate_up)
    check_training_dtype("swiglu", gate_up)
    return SwiGLUFunction.apply(gate_up)


def layernorm(x, weight, bias, eps):
    if not records(x, weight, bias):
        return ops.layernorm(x.contiguous(), weight, bias, eps)
    check_training_dtype("layernorm", x)
    return LayerNormFunction.apply(x, weight, bias, eps)


def attention_general(q, k, v, key_mask=None, scale=None):
    if not records(q, k, v):
        return ops.attention(q.contiguous(), k.contiguous(), v.contiguous(), key_mask=key_mask, scale=scale,
                             causal=False)
    check_training_dtype("attention_general", q)
    return GeneralAttentionFunction.apply(q, k, v, key_mask, float(scale if scale is not None else q.shape[-1] ** -0.5))


def quick_gelu(h):
    if not records(h):
        return h * torch.sigmoid(1.702 * h)
    check_training_dtype("quick_gelu", h)
    return QuickGELUFunction.apply(h)


def resize_bilinear(x, scale_factor):
    if not records(x):
        return F.interpolate(x, scale_factor=scale_factor, mode="bilinear", align_corners=False)
    check_training_dtype("resize_bilinear", x)
    return ResizeBilinearFunction.apply(x, scale_factor)


def conv(x, conv_module, add_bc=None, residual=None):
    if not records(x, residual, add_bc, conv_module):
        return conv_module.fused(x, add_bc, residual)
    return ConvFunction.apply(x, residual, conv_module, add_bc)


def group_norm_nhwc(x, groups, weight=None, bias=None, eps=1e-5, silu=False):
    if not records(x, weight, bias):
        return ops.group_norm_nhwc(x, groups, weight, bias, eps, silu=silu)
    return GroupNormNHWCFunction.apply(x, weight, bias, groups, float(eps), bool(silu))


def geglu(value_gate):
    if not records(value_gate):
        return ops.geglu(value_gate.contiguous())
    check_training_dtype("geglu", value_gate)
    return GEGLUFunction.apply(value_gate)
