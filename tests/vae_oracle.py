"""Independent fp32 restatement of diffusers 0.20.0's ``AutoencoderKL.decode`` (TEST INFRASTRUCTURE ONLY).

**Parity unpinned**, as for the UNet (oracle/unet.py): the arithmetic lives in diffusers, which is not installed here,
and the reference ships no fixture for it.  The reference's own part is the call (decoders/sd.py:212-216:
``vae.decode(latents / scaling_factor)``, then ``(x / 2 + 0.5).clamp(0, 1)``); the block algorithms restate diffusers'
published modules (autoencoder_kl.py, vae.py ``Decoder``, unet_2d_blocks.py ``UNetMidBlock2D`` / ``UpDecoderBlock2D``,
resnet.py, attention_processor.py).

Written against a flat state dict with diffusers' parameter names (``post_quant_conv.*``, ``decoder.*``); the block
structure is derived from the keys, and only torch.nn.functional ops are used, with oracle/unet.py's helpers.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.unet import _conv, _count, _lin

EPS = 1e-6          # every GroupNorm of the SD VAE


def resnet_ref(sd, p, x, groups=32, eps=EPS):
    """``ResnetBlock2D.forward`` with ``temb_channels=None``: GN -> SiLU -> conv1 -> GN -> SiLU -> conv2, 1x1
    ``conv_shortcut`` when the channel count changes, output_scale_factor 1."""
    h = F.silu(F.group_norm(x, groups, sd[p + ".norm1.weight"], sd[p + ".norm1.bias"], eps))
    h = _conv(sd, p + ".conv1", h)
    h = F.silu(F.group_norm(h, groups, sd[p + ".norm2.weight"], sd[p + ".norm2.bias"], eps))
    h = _conv(sd, p + ".conv2", h)
    if p + ".conv_shortcut.weight" in sd:
        x = _conv(sd, p + ".conv_shortcut", x, padding=0)
    return x + h


def attention_ref(sd, p, x, groups=32, eps=EPS):
    """``Attention`` of the VAE mid block (``_from_deprecated_attn_block``): GN -> one head over all channels with biased
    projections -> softmax(q k^T / sqrt(C)) -> to_out.0 -> + residual (``residual_connection=True``, rescale 1)."""
    B, C, H, W = x.shape
    h = F.group_norm(x, groups, sd[p + ".group_norm.weight"], sd[p + ".group_norm.bias"], eps)
    h = h.reshape(B, C, H * W).transpose(1, 2)
    q, k, v = _lin(sd, p + ".to_q", h), _lin(sd, p + ".to_k", h), _lin(sd, p + ".to_v", h)
    w = torch.softmax(torch.matmul(q, k.transpose(1, 2)) * C ** -0.5, dim=-1)
    o = _lin(sd, p + ".to_out.0", torch.matmul(w, v))
    return o.transpose(1, 2).reshape(B, C, H, W) + x


def vae_decode_ref(sd, z):
    """``AutoencoderKL.decode(z)`` (z already divided by the scaling factor): post_quant_conv (1x1) -> Decoder:
    conv_in -> mid block (resnet, attention, resnet) -> up blocks (resnets, then nearest 2x + 3x3 conv where an
    ``upsamplers`` entry exists) -> GroupNorm + SiLU -> conv_out.  fp32 CPU tensors; returns the image in [-1, 1]."""
    sd = {k: v.float() for k, v in sd.items()}
    x = _conv(sd, "post_quant_conv", z.float(), padding=0)
    x = _conv(sd, "decoder.conv_in", x)
    x = resnet_ref(sd, "decoder.mid_block.resnets.0", x)
    for i in range(_count(sd, "decoder.mid_block.", "attentions")):
        x = attention_ref(sd, f"decoder.mid_block.attentions.{i}", x)
        x = resnet_ref(sd, f"decoder.mid_block.resnets.{i + 1}", x)
    for b in range(_count(sd, "decoder.", "up_blocks")):
        p = f"decoder.up_blocks.{b}"
        for i in range(_count(sd, p + ".", "resnets")):
            x = resnet_ref(sd, f"{p}.resnets.{i}", x)
        if _count(sd, p + ".", "upsamplers") > 0:
            x = _conv(sd, f"{p}.upsamplers.0.conv", F.interpolate(x, scale_factor=2.0, mode="nearest"))
    x = F.silu(F.group_norm(x, 32, sd["decoder.conv_norm_out.weight"], sd["decoder.conv_norm_out.bias"], EPS))
    return _conv(sd, "decoder.conv_out", x)
