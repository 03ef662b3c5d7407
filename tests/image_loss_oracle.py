"""Independent restatements for the image-decoder loss (TEST INFRASTRUCTURE ONLY): the SD VAE's encode in fp32 and the
noise scheduler's forward-diffusion arithmetic in float64.

**Parity unpinned**, as for the decode (tests/vae_oracle.py): the arithmetic lives in diffusers 0.20.0, which is not
installed here.  The reference's own part is the call sequence (decoders/sd.py:220-316: ``vae.encode(x)
.latent_dist.sample() * scaling_factor``, ``noise_scheduler.add_noise`` / ``get_velocity``); the block algorithms
restate diffusers' published modules (autoencoder_kl.py ``encode``, vae.py ``Encoder`` / ``DiagonalGaussianDistribution``,
unet_2d_blocks.py ``DownEncoderBlock2D``, resnet.py ``Downsample2D``, scheduling_ddpm.py ``add_noise`` /
``get_velocity``).  Written against a flat state dict with diffusers' parameter names; the block structure is derived
from the keys, and only torch.nn.functional ops are used, with oracle/unet.py's helpers.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.unet import _conv, _count
from tests.vae_oracle import EPS, attention_ref, resnet_ref


def vae_encode_ref(sd, x):
    """``AutoencoderKL.encode(x).latent_dist`` as (mean, logvar): Encoder = conv_in -> down blocks (resnets, then
    ``F.pad(x, (0, 1, 0, 1))`` + 3x3 / stride-2 conv where a ``downsamplers`` entry exists) -> mid block (resnet,
    attention, resnet) -> GroupNorm + SiLU -> conv_out; then quant_conv (1x1); the moments split in two along the
    channels and the log-variance clamped to [-30, 20].  fp32 tensors in, fp32 out."""
    sd = {k: v.float() for k, v in sd.items()}
    x = _conv(sd, "encoder.conv_in", x.float())
    for b in range(_count(sd, "encoder.", "down_blocks")):
        p = f"encoder.down_blocks.{b}"
        for i in range(_count(sd, p + ".", "resnets")):
            x = resnet_ref(sd, f"{p}.resnets.{i}", x)
        if _count(sd, p + ".", "downsamplers") > 0:
            x = _conv(sd, f"{p}.downsamplers.0.conv", F.pad(x, (0, 1, 0, 1)), stride=2, padding=0)
    x = resnet_ref(sd, "encoder.mid_block.resnets.0", x)
    for i in range(_count(sd, "encoder.mid_block.", "attentions")):
        x = attention_ref(sd, f"encoder.mid_block.attentions.{i}", x)
        x = resnet_ref(sd, f"encoder.mid_block.resnets.{i + 1}", x)
    x = F.silu(F.group_norm(x, 32, sd["encoder.conv_norm_out.weight"], sd["encoder.conv_norm_out.bias"], EPS))
    moments = _conv(sd, "quant_conv", _conv(sd, "encoder.conv_out", x), padding=0)
    mean, logvar = moments.chunk(2, dim=1)
    return mean, logvar.clamp(-30.0, 20.0)


def _coefficients(alphas_cumprod, timesteps, ndim):
    a = alphas_cumprod.double()[timesteps.cpu()].view((-1,) + (1,) * (ndim - 1))
    return a.sqrt(), (1.0 - a).sqrt()


def add_noise_ref(alphas_cumprod, x, noise, timesteps):
    """``sqrt(abar_t) x + sqrt(1 - abar_t) eps`` in float64, abar_t = ``alphas_cumprod[t]`` of each sample as given (a
    caller restating a 16-bit sample passes the table rounded to that dtype, as diffusers rounds it)."""
    a, b = _coefficients(alphas_cumprod, timesteps, x.dim())
    return a * x.double().cpu() + b * noise.double().cpu()


def get_velocity_ref(alphas_cumprod, x, noise, timesteps):
    """``sqrt(abar_t) eps - sqrt(1 - abar_t) x`` in float64 (the v-prediction target)."""
    a, b = _coefficients(alphas_cumprod, timesteps, x.dim())
    return a * noise.double().cpu() - b * x.double().cpu()
