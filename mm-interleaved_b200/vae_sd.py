"""SD-2.1 VAE (``AutoencoderKL.decode`` and, optionally, ``encode``), H100-native assembly.

The reference decodes every generated image with diffusers 0.20.0's ``AutoencoderKL`` (decoders/sd.py:212-216:
``latents / scaling_factor``, ``vae.decode``, ``(x / 2 + 0.5).clamp(0, 1)``) and encodes the training / validation
images of the image-decoder loss with it (sd.py:220-238: ``vae.encode(x).latent_dist.sample() * scaling_factor``).
diffusers is not a dependency of this repository, so this file restates the published SD-2.1 VAE configuration (latent
channels 4, block_out_channels (128, 256, 512, 512), 2 layers per block, GroupNorm(32) with eps 1e-6, one single-head
attention over 512 channels in the mid blocks) with diffusers' parameter naming, so that a reference checkpoint's
``image_decoder.decoder.vae.*`` keys load one-to-one.  By default only the decoder half is built: ``post_quant_conv``
and ``decoder.*``; a full VAE state dict loads with ``strict=False`` and leaves ``encoder.*`` / ``quant_conv.*`` unused.
``with_encoder=True`` adds ``encoder.*`` and ``quant_conv``, and the full state dict loads with ``strict=True``.
**Parity is unpinned**, as for the UNet: the model-level checks are against the fp32 restatements in tests/vae_oracle.py
(decode) and tests/image_loss_oracle.py (encode).

H100 side, for a bf16 / f16 module: every 3x3 / 1x1 convolution with Cin % 64 == 0 runs in this repo's implicit-GEMM
wgmma kernel (csrc/conv_igemm_sm100.cu, Cout tile 128 for 128 / 256 / 512 channels) with the ResNet residual fused
into the epilogue; the three upsamplers (nearest 2x, then 3x3 conv) run as one fused phase-form kernel that never forms
the 4x-size upsampled map (ops.conv2d_up2x), and the encoder's three downsamplers (one-sided pad, then 3x3 / stride-2
conv) run in the same kernel with the pad taken from TMA's zero fill (ops.conv2d_down2x); GroupNorm(+SiLU) runs in the
NHWC kernel.  ``post_quant_conv`` / ``quant_conv``, the decoder's ``conv_in`` (Cin = 4) / ``conv_out`` (Cout = 3) and
the encoder's ``conv_in`` (Cin = 3) / ``conv_out`` (Cout = 8) stay on cuDNN, and the mid-block attention (one head of
512, T = HW of the latent, ~2 % of the decode's FLOPs, ~4 % of the encode's) runs as cuBLAS batched GEMMs around an
fp32 softmax.  An fp32 module runs on cuDNN / cuBLAS throughout (NCHW), which is the precision the reference decodes and
encodes in.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import ops, unet_sd
from .unet_sd import ResnetBlock2D, _gn

# attention parameter names of diffusers checkpoints saved before its Attention rename (AttentionBlock)
_DEPRECATED_ATTN_NAMES = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


class VAEAttention(nn.Module):
    """diffusers ``Attention`` as the VAE mid block builds it: GroupNorm(eps 1e-6) -> biased to_q / to_k / to_v over
    all channels as ONE head -> softmax(q k^T / sqrt(C)) in fp32 -> v -> ``to_out.0`` -> + residual."""

    def __init__(self, channels, groups=32, eps=1e-6):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, channels, eps=eps)
        self.to_q = nn.Linear(channels, channels)
        self.to_k = nn.Linear(channels, channels)
        self.to_v = nn.Linear(channels, channels)
        self.to_out = nn.ModuleList([nn.Linear(channels, channels), nn.Dropout(0.0)])

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        for old, new in _DEPRECATED_ATTN_NAMES.items():
            for suffix in ("weight", "bias"):
                key = f"{prefix}{old}.{suffix}"
                if key in state_dict:
                    state_dict[f"{prefix}{new}.{suffix}"] = state_dict.pop(key)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def forward(self, x):
        B, C, H, W = x.shape
        h = _gn(self.group_norm, x, False).permute(0, 2, 3, 1).reshape(B, H * W, C)
        q, k, v = self.to_q(h), self.to_k(h), self.to_v(h)
        s = torch.baddbmm(q.new_zeros(1, 1, 1), q, k.transpose(1, 2), beta=0, alpha=C ** -0.5)
        p = torch.softmax(s, dim=-1, dtype=torch.float32).to(q.dtype)
        o = self.to_out[0](torch.bmm(p, v))
        return o.reshape(B, H, W, C).permute(0, 3, 1, 2) + x


class Upsample2D(unet_sd.Upsample2D):
    """Nearest 2x + 3x3 conv; on the fused phase-form kernel when the layer qualifies (ops.conv2d_up2x_supported),
    else ``conv(interpolate(x))`` as in the UNet."""

    def forward(self, x):
        w = self.conv.weight
        if unet_sd.USE_CONV_KERNEL and x.is_contiguous(memory_format=torch.channels_last) and ops.conv2d_up2x_supported(x, w):
            return ops.conv2d_up2x(x, self.conv.weight_up2x(), self.conv.bias)
        return super().forward(x)


class Downsample2D(nn.Module):
    """diffusers ``Downsample2D(padding=0)`` of the encoder: ``conv3x3(F.pad(x, (0, 1, 0, 1)), stride 2)``; in one kernel
    without the padded copy when the layer qualifies (ops.conv2d_down2x_supported), else pad + the library convolution."""

    def __init__(self, channels):
        super().__init__()
        self.conv = unet_sd.Conv2d(channels, channels, 3, stride=2, padding=0)

    def forward(self, x):
        w = self.conv.weight
        if unet_sd.USE_CONV_KERNEL and x.is_contiguous(memory_format=torch.channels_last) and ops.conv2d_down2x_supported(x, w):
            return ops.conv2d_down2x(x, self.conv.weight_khwc(), self.conv.bias)
        return self.conv(F.pad(x, (0, 1, 0, 1)))


class UNetMidBlock2D(nn.Module):
    def __init__(self, channels, groups=32, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(channels, channels, None, groups, eps) for _ in range(2)])
        self.attentions = nn.ModuleList([VAEAttention(channels, groups, eps)])

    def forward(self, x):
        x = self.resnets[0](x)
        return self.resnets[1](self.attentions[0](x))


class UpDecoderBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, layers, add_upsample, groups=32, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(in_channels if i == 0 else out_channels, out_channels, None, groups, eps)
                                      for i in range(layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(out_channels)]) if add_upsample else None

    def forward(self, x):
        for res in self.resnets:
            x = res(x)
        return x if self.upsamplers is None else self.upsamplers[0](x)


class Decoder(nn.Module):
    """diffusers ``Decoder``: conv_in -> mid block -> up blocks over the reversed ``block_out_channels`` (each
    ``layers_per_block + 1`` resnets, an upsampler on all but the last) -> GroupNorm + SiLU -> conv_out."""

    def __init__(self, in_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 norm_num_groups=32):
        super().__init__()
        rev = list(reversed(block_out_channels))
        self.conv_in = nn.Conv2d(in_channels, rev[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(rev[0], norm_num_groups)
        self.up_blocks = nn.ModuleList()
        prev = rev[0]
        for i, ch in enumerate(rev):
            self.up_blocks.append(UpDecoderBlock2D(prev, ch, layers_per_block + 1, i != len(rev) - 1, norm_num_groups))
            prev = ch
        self.conv_norm_out = nn.GroupNorm(norm_num_groups, rev[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(rev[-1], out_channels, 3, padding=1)

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        for blk in self.up_blocks:
            x = blk(x)
        return self.conv_out(_gn(self.conv_norm_out, x, True))


class DownEncoderBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, layers, add_downsample, groups=32, eps=1e-6):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(in_channels if i == 0 else out_channels, out_channels, None, groups, eps)
                                      for i in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(out_channels)]) if add_downsample else None

    def forward(self, x):
        for res in self.resnets:
            x = res(x)
        return x if self.downsamplers is None else self.downsamplers[0](x)


class Encoder(nn.Module):
    """diffusers ``Encoder`` (``double_z=True``): conv_in -> down blocks over ``block_out_channels`` (each
    ``layers_per_block`` resnets, a padding-0 downsampler on all but the last) -> mid block -> GroupNorm + SiLU ->
    conv_out to 2 x ``out_channels`` (the posterior's mean and log-variance)."""

    def __init__(self, in_channels=3, out_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 norm_num_groups=32):
        super().__init__()
        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], 3, padding=1)
        self.down_blocks = nn.ModuleList()
        prev = block_out_channels[0]
        for i, ch in enumerate(block_out_channels):
            self.down_blocks.append(DownEncoderBlock2D(prev, ch, layers_per_block, i != len(block_out_channels) - 1,
                                                       norm_num_groups))
            prev = ch
        self.mid_block = UNetMidBlock2D(block_out_channels[-1], norm_num_groups)
        self.conv_norm_out = nn.GroupNorm(norm_num_groups, block_out_channels[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(block_out_channels[-1], 2 * out_channels, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for blk in self.down_blocks:
            x = blk(x)
        return self.conv_out(_gn(self.conv_norm_out, self.mid_block(x), True))


class DiagonalGaussianDistribution:
    """diffusers' posterior of ``AutoencoderKL.encode``: the moments (B, 2 C, h, w) split into ``mean`` and ``logvar``
    (clamped to [-30, 20]); ``std = exp(logvar / 2)``."""

    def __init__(self, parameters: torch.Tensor):
        self.parameters = parameters
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """``mean + std * eps``, eps standard normal in the moments' dtype, drawn from ``generator`` (else the global
        generator of the moments' device)."""
        eps = torch.randn(self.mean.shape, generator=generator, device=self.parameters.device, dtype=self.parameters.dtype)
        return self.mean + self.std * eps

    def mode(self) -> torch.Tensor:
        return self.mean


class AutoencoderKLOutput:
    """What ``AutoencoderKL.encode`` returns, as in diffusers: ``.latent_dist``."""

    __slots__ = ("latent_dist",)

    def __init__(self, latent_dist: DiagonalGaussianDistribution):
        self.latent_dist = latent_dist


class AutoencoderKL(nn.Module):
    """diffusers' ``AutoencoderKL`` with the SD-2.1 configuration as defaults.  By default only the decoder half
    (``post_quant_conv``, ``decoder``: 49.49 M parameters); ``with_encoder=True`` also builds ``encoder`` and
    ``quant_conv`` (34.16 M more), and a full VAE state dict then loads with ``strict=True``.  The encoder reads images
    with ``out_channels`` channels, the ones the decoder writes."""

    def __init__(self, latent_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 norm_num_groups=32, scaling_factor=0.18215, with_encoder=False):
        super().__init__()
        self.scaling_factor = scaling_factor
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
        self.decoder = Decoder(latent_channels, out_channels, block_out_channels, layers_per_block, norm_num_groups)
        self.encoder = self.quant_conv = None
        if with_encoder:       # built after the decoder: the same seed gives the same decoder weights either way
            self.encoder = Encoder(out_channels, latent_channels, block_out_channels, layers_per_block, norm_num_groups)
            self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)

    @torch.no_grad()
    def encode(self, x: torch.Tensor) -> AutoencoderKLOutput:
        """Image (B, 3, H, W) in [-1, 1] to the posterior over the latents (B, 4, H/8, W/8), in the module's dtype:
        ``encode(x).latent_dist.sample()`` as diffusers.  A 16-bit module on the GPU runs channels_last."""
        if self.encoder is None:
            raise RuntimeError("AutoencoderKL.encode: this VAE has no encoder (build it with with_encoder=True)")
        w = self.quant_conv.weight
        x = x.to(device=w.device, dtype=w.dtype)
        if x.is_cuda and w.dtype in (torch.bfloat16, torch.float16):
            x = x.contiguous(memory_format=torch.channels_last)
        return AutoencoderKLOutput(DiagonalGaussianDistribution(self.quant_conv(self.encoder(x))))

    @torch.no_grad()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """Latents (B, 4, h, w) -- already divided by ``scaling_factor`` -- to the image (B, 3, 8h, 8w) in [-1, 1], in
        the module's dtype.  A 16-bit module on the GPU runs channels_last, the layout the kernels read."""
        w = self.post_quant_conv.weight
        z = z.to(device=w.device, dtype=w.dtype)
        if z.is_cuda and w.dtype in (torch.bfloat16, torch.float16):
            z = z.contiguous(memory_format=torch.channels_last)
        return self.decoder(self.post_quant_conv(z))

    forward = decode
