"""Top-level glue of the interleaved forward: embed splice, image-visibility mask, MMFS feature
packing, decoder prefill and text head -- the body of ``MMInterleaved.forward`` up to the logits
(mm_interleaved/models/mm_interleaved.py:121-252, 408-455) and ``TextDecoder.forward``
(models/decoders/decoder_text.py:140-163).

Same semantics as the reference helpers, but written for the device: no Python loops over the batch,
no ``.nonzero()`` / ``.max()`` host synchronisations, no per-sample slicing -- everything is a handful
of tensor ops whose shapes are known from the (static) maximum image count.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.nn.functional as F
from torch import nn

from . import generation
from ._cache import WeightCache
from .llama_mmfs import LlamaMMFSConfig, LlamaModel
from .msda import records

# special-token convention of the reference (mm_interleaved.py:33-39; custom_datasets/wds_utils.py:186-215 appends
# "<|beginofimage|>" = 32000 and "<|image|>" = 32001 to the 32000 Llama ids)
DEFAULT_SPECIAL_TOKENS = dict(bos_token_id=1, eos_token_id=2, pad_token_id=31999, soi_token_id=32000, image_token_id=32001)


def splice_image_embeds(text_embeds, text_ids, image_embeds, soi_token, image_token_id, soi_token_id):
    """Steps 3 of ``_prepare_mm_embeds`` (mm_interleaved.py:144-170): the k-th ``<image>`` slot (row-major over the
    batch) receives the k-th row of ``image_embeds``; the learnable ``soi_token`` is added at every ``<soi>``."""
    is_img = (text_ids == image_token_id).unsqueeze(-1)
    out = text_embeds.to(image_embeds.dtype).masked_scatter(is_img, image_embeds.reshape(-1, image_embeds.shape[-1]))
    is_soi = (text_ids == soi_token_id).unsqueeze(-1).to(out.dtype)
    return out + is_soi * soi_token.to(out.dtype).view(1, 1, -1)


def cross_attention_mask_from_ids(text_ids, max_num_image: int, bos_token_id: int, soi_token_id: int,
                                  num_image_per_seq: Optional[torch.Tensor] = None):
    """(B, L, N) float 0/1: image n of a sequence is visible to token t iff ``soi_n + 1 > nearest_bos(t)`` and
    ``soi_n + 1 <= t`` (mm_interleaved.py:192-221).  Slots past a sequence's image count are never visible."""
    B, L = text_ids.shape
    ar = torch.arange(L, device=text_ids.device)
    soi_pos = torch.where(text_ids == soi_token_id, ar[None, :], L + 1).sort(dim=1).values[:, :max_num_image]
    if soi_pos.shape[1] < max_num_image:
        soi_pos = torch.nn.functional.pad(soi_pos, (0, max_num_image - soi_pos.shape[1]), value=L + 1)
    valid = soi_pos <= L
    if num_image_per_seq is not None:
        valid = valid & (torch.arange(max_num_image, device=text_ids.device)[None, :] < num_image_per_seq[:, None])
    img_pos = torch.where(valid, soi_pos + 1, torch.full_like(soi_pos, -1))            # (B, N)
    nearest_bos = torch.where(text_ids == bos_token_id, ar[None, :], -1).cummax(dim=1).values   # (B, L)
    vis = (img_pos[:, None, :] > nearest_bos[:, :, None]) & (img_pos[:, None, :] <= ar[None, :, None]) & \
          (img_pos[:, None, :] != -1)
    return vis.float()


def pack_mmfs_features(multiscale_features: Sequence[torch.Tensor], spatial_shapes: Sequence[int],
                       num_image_per_seq: torch.Tensor, max_num_image: int):
    """(B, N, sum(h*w), C): the maps whose side is in ``spatial_shapes``, zero-padded per sequence to ``max_num_image``
    images and flattened level by level (mm_interleaved.py:223-250)."""
    feats = [f for f in multiscale_features if int(f.shape[-1]) in spatial_shapes]
    B = num_image_per_seq.shape[0]
    first = torch.cumsum(num_image_per_seq, 0) - num_image_per_seq                      # first image of each sequence
    n_tot = feats[0].shape[0]
    img = torch.arange(n_tot, device=feats[0].device)
    seq_of = torch.bucketize(img, torch.cumsum(num_image_per_seq, 0), right=True)
    dest = seq_of * max_num_image + (img - first[seq_of])
    packed = []
    for f in feats:
        n, c, h, w = f.shape
        flat = f.flatten(2).transpose(1, 2)                                              # (n, hw, C)
        buf = flat.new_zeros((B * max_num_image, h * w, c))
        buf.index_copy_(0, dest, flat)
        packed.append(buf.view(B, max_num_image, h * w, c))
    return torch.cat(packed, dim=2)


def sincos_pos_embed_1d(embed_dim: int, length: int) -> torch.Tensor:
    """(length, embed_dim) [sin | cos] table of ``get_1d_sincos_pos_embed_from_grid`` (utils/pos_embed.py:77-95) for
    positions 0..length-1 (float32 arithmetic like the numpy original)."""
    import numpy as np
    omega = np.arange(embed_dim // 2, dtype=np.float32)
    omega /= embed_dim / 2.0
    omega = 1.0 / 10000 ** omega
    out = np.einsum("m,d->md", np.arange(length, dtype=np.float32), omega)
    return torch.from_numpy(np.concatenate([np.sin(out), np.cos(out)], axis=1))


def soi_positions(text_ids: torch.Tensor, soi_token_id: int, n_images: int):
    """Row / column of the first ``n_images`` ``<soi>`` tokens in row-major order, without ``nonzero`` (no host sync:
    the image count is known from the image tensor)."""
    B, L = text_ids.shape
    flat = torch.where((text_ids == soi_token_id).reshape(-1), torch.arange(B * L, device=text_ids.device), B * L)
    flat = flat.sort().values[:n_images]
    return flat // L, flat % L


def context_features_for_image_decoder(context_features: torch.Tensor, text_ids: torch.Tensor, soi_token_id: int,
                                       context_feat_proj: nn.Module, seq_len: int, n_images: int,
                                       nearest_bos_idxs: Optional[torch.Tensor] = None, pad_to: Optional[int] = None):
    """``_prepare_context_features_for_image_decoder`` (mm_interleaved.py:254-304): for every image, the decoder hidden
    states from its nearest ``<bos>`` (default: position 0) up to and including its ``<soi>``, in REVERSED order (the
    ``<soi>`` state first), zero-padded to the longest context, through ``context_feat_proj`` (padding rows included,
    as in the reference) plus the 1-D sin-cos table.  Returns (features (B_I, L_max, C), mask (B_I, L_max) int64).
    ``pad_to`` fixes L_max (no host sync); None reproduces the reference's data-dependent ``max(context_lengths)``."""
    rows, cols = soi_positions(text_ids, soi_token_id, n_images)
    bos = torch.zeros_like(cols) if nearest_bos_idxs is None else nearest_bos_idxs.to(cols.dtype)
    lengths = cols - bos + 1
    L_max = int(lengths.max()) if pad_to is None else int(pad_to)
    t = torch.arange(L_max, device=text_ids.device)
    src = cols[:, None] - t[None, :]                                   # reversed walk from the <soi> position
    valid = t[None, :] < lengths[:, None]
    gathered = context_features[rows[:, None], src.clamp(min=0)]       # (B_I, L_max, C)
    per_image = torch.where(valid[..., None], gathered, torch.zeros((), dtype=gathered.dtype, device=gathered.device))
    pos = sincos_pos_embed_1d(context_features.shape[-1], seq_len).to(device=per_image.device, dtype=per_image.dtype)
    per_image = context_feat_proj(per_image) + pos[None, :L_max]
    return per_image, valid.to(cols.dtype)


def mmfs_features_for_image_decoder(multiscale_features: Sequence[torch.Tensor], text_ids: torch.Tensor, soi_token_id: int,
                                    nearest_bos_idxs: Optional[torch.Tensor] = None):
    """``_prepare_mmfs_features_for_image_decoder`` (mm_interleaved.py:306-340): the tril/triu pair keeps exactly one
    candidate per image -- the image right before it in row-major order -- and it is used iff its ``<soi>`` lies at or
    after the current image's context start (``row * L + nearest_bos``).  Returns ([ (B_I, 1, C, h, w) ], (B_I, 1))."""
    n = multiscale_features[0].shape[0]
    L = text_ids.shape[1]
    rows, cols = soi_positions(text_ids, soi_token_id, n)
    start = rows * L + (torch.zeros_like(cols) if nearest_bos_idxs is None else nearest_bos_idxs.to(cols.dtype))
    flat = rows * L + cols
    prev = torch.arange(n, device=text_ids.device) - 1
    use = (prev >= 0) & (start <= flat[prev.clamp(min=0)])             # image_context_mask[i, i-1]
    feats = []
    for f in multiscale_features:
        g = f[prev.clamp(min=0)] * use.view(-1, 1, 1, 1).to(f.dtype)
        feats.append(g[:, None])
    return feats, use.to(torch.long)[:, None]


class TextDecoder(nn.Module):
    """``TextDecoder`` (decoders/decoder_text.py:26-163): ``head`` over the whole vocabulary plus ``head_new`` for the
    added ids, summed on the tail columns (:155-157); both carry a bias (:43-46).  State-dict names match the reference.
    ``forward`` keeps the reference signature (``inputs_embeds`` first, ``return_dict``); ``logits()`` is the plain
    tensor-in / tensor-out form used inside this package."""

    def __init__(self, hidden_size: int = None, vocab_size: int = 32002, orig_vocab_size: int = 32000, config=None,
                 txt_vocab_size: int = None, orig_txt_vocab_size: int = None, **_):
        super().__init__()
        if config is not None and hidden_size is None:                  # reference keyword form (decoder_text.py:27-34)
            hidden_size = config.hidden_size
        vocab_size = txt_vocab_size if txt_vocab_size is not None else vocab_size
        orig_vocab_size = orig_txt_vocab_size if orig_txt_vocab_size is not None else orig_vocab_size
        assert 0 < orig_vocab_size < vocab_size
        self.config = config
        self.orig_txt_vocab_size = orig_vocab_size
        self.head = nn.Linear(hidden_size, vocab_size, bias=True)
        self.head_new = nn.Linear(hidden_size, vocab_size - orig_vocab_size, bias=True)
        self._fused_cache = WeightCache()

    _PAD = 128   # a vocabulary of 32002+ rows is not a multiple of 8: cuBLAS drops to an unaligned legacy kernel (5x slower)

    def _fused(self):
        """head + head_new folded into one matrix / bias, rows zero-padded to a multiple of 128 (inference only)."""
        head, new = self.head, self.head_new
        return self._fused_cache.get((head.weight, new.weight, head.bias, new.bias), self._fold_heads)

    def _fold_heads(self):
        V, C = self.head.weight.shape
        Vp = (V + self._PAD - 1) // self._PAD * self._PAD
        w = self.head.weight.new_zeros((Vp, C))
        w[:V] = self.head.weight
        w[self.orig_txt_vocab_size:V] += self.head_new.weight
        b = self.head.bias.new_zeros((Vp,))
        b[:V] = self.head.bias
        b[self.orig_txt_vocab_size:V] += self.head_new.bias
        return w, b

    def logits(self, hidden_states):
        if records(self):
            logits = self.head(hidden_states)                                              # :155-157 as written
            tail = logits[..., self.orig_txt_vocab_size:] + self.head_new(hidden_states)
            return torch.cat([logits[..., :self.orig_txt_vocab_size], tail], dim=-1)
        w, b = self._fused()
        return F.linear(hidden_states, w, b)[..., :self.head.weight.shape[0]]

    def forward(self, inputs_embeds, attention_mask=None, position_ids=None, past_key_values=None, use_cache=None,
                output_attentions=None, output_hidden_states=None, return_dict=None, **kwargs):
        logits = self.logits(inputs_embeds)
        if not return_dict:
            return (logits,)
        from types import SimpleNamespace
        return SimpleNamespace(logits=logits, last_hidden_state=None, past_key_values=None, hidden_states=None,
                               attentions=None)


TextHead = TextDecoder   # round-1 name


class StableDiffusion(nn.Module):
    """``StableDiffusion`` (decoders/sd.py:23-218) on this repo's modules: ``unet`` (SD-2.1-base UNet with the patched
    forward, unet_sd.py), ``mmfs_module`` (MMFSNet) and ``noise_scheduler`` (scheduler.py: DDPM on the SD-2.1-base
    schedule, sd.py:48-50) -- same attribute / state-dict names as the reference.  ``vae`` (e.g. the SD-2.1 decoder
    ``vae_sd.AutoencoderKL``) is registered as ``self.vae`` -- state-dict keys ``vae.*`` as in a reference checkpoint --
    and ``vae_decode`` defaults to its ``decode``; any callable latents -> image in [-1, 1] may be given as
    ``vae_decode`` instead.  Without either, ``generate_images`` returns the denoised latents (the pipeline's
    ``output_type="latent"`` result, sd.py:196-211).  ``forward`` (the denoising loss) needs a VAE with an encoder
    (``vae_sd.AutoencoderKL(with_encoder=True)``); it encodes in chunks of ``vae_encode_mini_bs`` images (<= 0: one
    chunk)."""

    def __init__(self, unet=None, mmfs_module=None, image_size=512, base_seed=0, use_random_seed=False,
                 noise_scheduler=None, vae_decode=None, vae_scaling_factor=0.18215, vae=None, vae_encode_mini_bs=32,
                 **unet_kwargs):
        super().__init__()
        from . import unet_sd
        from .scheduler import DDPMScheduler, SD21_BASE_SCHEDULER
        self.unet = unet if unet is not None else unet_sd.UNet2DConditionModel(**unet_kwargs)
        self.mmfs_module = mmfs_module
        self.image_size, self.base_seed, self.use_random_seed = image_size, base_seed, use_random_seed
        self.vae_encode_mini_bs = vae_encode_mini_bs
        self.noise_scheduler = noise_scheduler if noise_scheduler is not None else DDPMScheduler(**SD21_BASE_SCHEDULER)
        self.vae = vae
        if vae is not None and vae_decode is None:
            vae_decode = vae.decode
        self.vae_decode, self.vae_scaling_factor = vae_decode, vae_scaling_factor
        self._unet_graphs = None        # enable_cuda_graphs(): {input shapes -> unet_sd.GraphedUNet}, kept across calls

    def enable_cuda_graphs(self, on: bool = True):
        """Replay the UNet evaluation (~1200 kernels) from a CUDA graph captured once per input shape and kept across
        ``generate_images`` calls (SURVEY.md 8 f3); the per-call MMFS image-side state is refreshed in place."""
        self._unet_graphs = {} if on else None
        return self

    @torch.no_grad()
    def generate_images(self, text_embeds, negative_prompt_embeds=None, num_validation_images=1, num_inference_steps=30,
                        mini_bs=8, guidance_scale=7.5, mmfs_features=None, mmfs_mask=None, latents=None):
        """sd.py:142-218: per validation image one generator seeded ``base_seed + num`` that draws the initial latents
        AND the scheduler noise of every mini-batch in turn; mini-batches of ``mini_bs`` prompts through the CFG loop."""
        import math
        import numpy as np
        from .unet_sd import denoise_loop
        side = self.image_size // 8
        outs = []
        for num in range(num_validation_images):
            seed = num + (int(np.random.randint(self.base_seed)) if self.use_random_seed else self.base_seed)
            gen = torch.Generator(device=text_embeds.device).manual_seed(seed)
            for it in range(math.ceil(text_embeds.shape[0] / mini_bs)):
                sl = slice(it * mini_bs, it * mini_bs + mini_bs)
                txt = text_embeds[sl]
                neg = negative_prompt_embeds[sl] if negative_prompt_embeds is not None else torch.zeros_like(txt)
                if latents is not None:
                    lat = latents[sl]
                else:
                    lat = torch.randn((txt.shape[0], 4, side, side), generator=gen, device=txt.device, dtype=txt.dtype)
                if lat.is_cuda:
                    lat = lat.contiguous(memory_format=torch.channels_last)
                lat = denoise_loop(self.unet, lat, txt, neg,
                                   [f[sl] for f in mmfs_features] if mmfs_features is not None else None,
                                   mmfs_mask[sl] if mmfs_mask is not None else None, self.mmfs_module,
                                   num_steps=num_inference_steps, guidance=guidance_scale, scheduler=self.noise_scheduler,
                                   generator=gen, graph_cache=self._unet_graphs)
                outs.append(lat)
        lat = torch.cat(outs, dim=0)
        if self.vae_decode is None:
            return lat
        image = self.vae_decode(lat.float() / self.vae_scaling_factor)                       # sd.py:212-215
        return (image / 2 + 0.5).clamp(0, 1).float()

    def _encode_latents(self, image, dtype, generator=None):
        """sd.py:220-238: posterior samples of ``vae_encode_mini_bs`` images at a time, cast to ``dtype``, times the
        scaling factor.  The VAE encodes in its own dtype (the reference casts it to fp32), under ``torch.no_grad()`` as
        there: the VAE is frozen and nothing upstream of the latents trains."""
        n = self.vae_encode_mini_bs if self.vae_encode_mini_bs > 0 else image.shape[0]
        with torch.no_grad():
            parts = [self.vae.encode(image[i:i + n]).latent_dist.sample(generator).to(dtype)
                     for i in range(0, image.shape[0], n)]
        return torch.cat(parts, dim=0) * self.vae_scaling_factor

    def forward(self, image, text_embeds, return_outputs=False, mmfs_features=None, mmfs_mask=None,
                generator: Optional[torch.Generator] = None):
        """The denoising loss of sd.py:240-316.  Under autograd its gradient reaches ``text_embeds``, the MMFS hook
        (``mmfs_module``) and ``mmfs_features`` through the frozen UNet (``unet.requires_grad_(False)``; the UNet's own
        weights have no backward here).  ``image`` (B, 3, S, S) in [0, 1] with S = ``image_size``; returns the per-element
        ``mse(unet(noisy, t), target)`` in fp32, shaped like the latents, or with ``return_outputs`` the reference's
        ``dict(loss, pred, target)`` plus ``latents`` and ``timesteps``.

        Random draws, in this order: the posterior noise of each encode chunk, the diffusion noise (like the latents, in
        the UNet's dtype), one timestep in [0, num_train_timesteps) per image -- from ``generator`` when given, else from
        the global generator, as the reference does.  Differences from the reference: the image is normalised out of
        place (the reference's ``image.sub_(0.5).div_(0.5)`` rewrites the caller's tensor), and the UNet runs eagerly on
        the (B,) timesteps with no classifier-free-guidance batch."""
        h, w = image.shape[-2:]
        assert h == self.image_size and w == self.image_size, f"{tuple(image.shape)=} {self.image_size=}"
        if getattr(self.vae, "encoder", None) is None:
            raise RuntimeError("StableDiffusion.forward needs a VAE with an encoder (vae_sd.AutoencoderKL(with_encoder=True))")
        dtype = next(self.unet.parameters()).dtype
        latents = self._encode_latents((image - 0.5) / 0.5, dtype, generator)
        noise = torch.randn(latents.shape, generator=generator, device=latents.device, dtype=latents.dtype)
        timesteps = torch.randint(0, self.noise_scheduler.num_train_timesteps, (latents.shape[0],), generator=generator,
                                  device=latents.device)
        noisy = self.noise_scheduler.add_noise(latents, noise, timesteps)
        pt = self.noise_scheduler.prediction_type
        if pt == "epsilon":
            target = noise
        elif pt == "v_prediction":
            target = self.noise_scheduler.get_velocity(latents, noise, timesteps)
        else:
            raise ValueError(f"Unknown prediction type {pt}")
        if noisy.is_cuda:
            noisy = noisy.contiguous(memory_format=torch.channels_last)
        pred = self.unet(noisy, timesteps, text_embeds, mmfs_features=mmfs_features, mmfs_mask=mmfs_mask,
                         mmfs_module=self.mmfs_module)
        loss = F.mse_loss(pred.float(), target.float(), reduction="none")
        if not return_outputs:
            return loss
        return dict(loss=loss, pred=pred, target=target, latents=latents, timesteps=timesteps)


class ImageDecoder(nn.Module):
    """``ImageDecoder`` (decoders/decoder_image.py:9-156): ``perceiver_resampler`` (Q-Former, 77 queries of width 1024
    over the per-image LLM context), ``neg_prompt_embeds`` and ``decoder`` = ``StableDiffusion`` (UNet + MMFSNet +
    scheduler, and the VAE decoder when ``vae`` is given).  State-dict names follow the reference (``decoder.unet.*``,
    ``decoder.mmfs_module.*``, ``decoder.vae.*``).  ``vae``: ``True`` builds the SD-2.1 decoder (vae_sd.py), a dict
    builds ``vae_sd.AutoencoderKL(**vae)`` (``{"with_encoder": True}`` adds the encoder that ``forward``, the image
    loss, needs), a module is used as it is; it applies when ``decoder`` is not given."""

    def __init__(self, perceiver_config=None, seq_len=77, embed_dim=1024, unet=None, mmfs_module=None, image_size=512,
                 base_seed=0, sd_base_seed=None, sd_use_random_seed=False, mmfs_input_channel=1024, mmfs_feat_levels=4,
                 uncond_prob=0.1, decoder: Optional[nn.Module] = None, vae=None, vae_encode_mini_bs=32, **_):
        super().__init__()
        from .visual_tokenizer import PerceiverResampler
        self.uncond_prob = uncond_prob
        self.perceiver_resampler = PerceiverResampler(**(perceiver_config or dict(num_queries=seq_len, hidden_size=embed_dim)))
        self.neg_prompt_embeds = nn.Parameter(torch.zeros(1, seq_len, embed_dim).normal_(0, 0.02))
        if decoder is None:
            if unet is None:            # full-size SD-2.1-base UNet + its MMFSNet (sd.py:58-82)
                from . import unet_sd
                from .sd_mmfs import MMFSNet
                unet = unet_sd.UNet2DConditionModel()
                mmfs_module = MMFSNet(mmfs_input_channel, tuple(unet.block_out_channels), 2,
                                      downsample_factor=512 // image_size, n_levels=mmfs_feat_levels)
            if vae is True or isinstance(vae, dict):
                from .vae_sd import AutoencoderKL
                vae = AutoencoderKL(**(vae if isinstance(vae, dict) else {}))
            decoder = StableDiffusion(unet=unet, mmfs_module=mmfs_module, image_size=image_size,
                                      base_seed=base_seed if sd_base_seed is None else sd_base_seed,
                                      use_random_seed=sd_use_random_seed, vae=None if vae is False else vae,
                                      vae_encode_mini_bs=vae_encode_mini_bs)
        self.decoder = decoder

    # round-1 attribute names
    unet = property(lambda self: self.decoder.unet)
    mmfs_module = property(lambda self: self.decoder.mmfs_module)

    def forward(self, image_tensors, context_features, context_attention_mask=None, image_loss_mask=None,
                mmfs_features=None, mmfs_mask=None, generator: Optional[torch.Generator] = None):
        """decoder_image.py:69-120: the image loss of B_I images, a scalar.  Q-Former over the per-image context; with
        probability ``uncond_prob`` an image's prompt is replaced by ``neg_prompt_embeds`` (in eval mode too, as in the
        reference; that ``rand`` is drawn before the diffusion loss's draws, from ``generator`` when given); the
        per-element SD loss is zeroed for images whose context has <= 2 tokens (``<bos>``, ``<soi>``) and where
        ``image_loss_mask`` is 0, then averaged over every element, zeroed ones included.  Differentiable: under
        autograd the gradient reaches the Q-Former, ``neg_prompt_embeds``, the MMFS hook, ``context_features`` and
        ``mmfs_features`` through the frozen UNet (``decoder.unet.requires_grad_(False)``; its own weights have no
        backward here)."""
        assert image_tensors.shape[0] == context_features.shape[0]
        if context_attention_mask is None:
            raise ValueError("ImageDecoder.forward needs context_attention_mask")
        assert bool(torch.all(context_attention_mask.sum(dim=1) > 0)), "an image has an empty context"
        ctx = self.perceiver_resampler(encoder_hidden_states=context_features,
                                       encoder_attention_mask=context_attention_mask)[0]
        if self.uncond_prob > 0.0:
            u = torch.rand(ctx[:, :1, :1].shape, generator=generator, device=ctx.device, dtype=ctx.dtype)
            ctx = torch.where(u < self.uncond_prob, self.neg_prompt_embeds.to(ctx.dtype), ctx)
        loss = self.decoder(image_tensors, ctx, mmfs_features=mmfs_features, mmfs_mask=mmfs_mask, generator=generator)
        loss = loss * (context_attention_mask.sum(dim=1) > 2).to(loss.device).view(-1, 1, 1, 1)
        if image_loss_mask is not None:
            loss = loss * image_loss_mask.to(loss.device).view(-1, 1, 1, 1)
        return loss.mean()

    @torch.no_grad()
    def generate_images(self, context_features, context_attention_mask=None, mmfs_features=None, mmfs_mask=None, **kwargs):
        """decoder_image.py:122-156.  Returns ``{"image": ...}`` (decoded images when the decoder has a VAE, else the
        latents) and always ``{"latents": ...}`` when no VAE is attached."""
        text_embeds = self.perceiver_resampler(encoder_hidden_states=context_features,
                                               encoder_attention_mask=context_attention_mask)[0]        # :132-136
        num_inference_steps = kwargs.pop("num_inference_steps", 30)
        guidance_scale = kwargs.pop("guidance_scale", 7.5)
        num_validation_images = kwargs.pop("num_validation_images", 1)
        neg = self.neg_prompt_embeds.to(text_embeds.dtype).expand_as(text_embeds)                       # :141-143
        res = self.decoder.generate_images(text_embeds=text_embeds, negative_prompt_embeds=neg,
                                           num_validation_images=num_validation_images,
                                           num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                                           mmfs_features=mmfs_features, mmfs_mask=mmfs_mask,
                                           latents=kwargs.pop("latents", None))
        out = {"image": res}
        if self.decoder.vae_decode is None:
            out["latents"] = res
        return out


class InterleavedForward(nn.Module):
    """``mm_decoder`` + ``text_decoder`` + ``soi_token`` of ``MMInterleaved`` with the forward path of
    ``MMInterleaved.forward`` up to the text logits.  Image embeddings / multi-scale maps come from the visual
    tokenizer (``visual_output`` dict with ``vis_embed`` and ``multiscale_features``, visual_tokenizer.py:96-101)."""

    def __init__(self, config: LlamaMMFSConfig, special_tokens=None, orig_vocab_size: int = 32000, seq_len: int = 2048,
                 image_decoder: Optional[nn.Module] = None):
        super().__init__()
        self.config = config
        self.special_token_dict = dict(DEFAULT_SPECIAL_TOKENS if special_tokens is None else special_tokens)
        self.mm_decoder = LlamaModel(config)
        self.text_decoder = TextDecoder(config.hidden_size, config.vocab_size, orig_vocab_size)
        self.soi_token = nn.Parameter(torch.zeros(1, config.hidden_size))
        self.spatial_shapes = list(config.spatial_shapes)
        self.context_feat_proj = nn.Linear(config.hidden_size, config.hidden_size)       # mm_interleaved.py:99
        self.seq_len = seq_len
        self.image_decoder = image_decoder                                                # ImageDecoder or None
        self._decode_graphs = None                                                        # enable_decode_graphs()
        self._decode_graph_sampling = False

    def enable_decode_graphs(self, enabled: bool = True, sampling: bool = False) -> "InterleavedForward":
        """Greedy ``generate_texts`` then replays ONE captured CUDA graph per generated token (embedding -> 40 layers ->
        head -> logits processors -> arg-max -> state update, ~1000 kernels) instead of launching them from Python; the
        graph, its static KV cache and input buffers are kept per (batch, cache length, image count) and reused by
        later calls (SURVEY.md 8 f3; causal_lm_cascade.py:171-204 is the loop it replaces).  The token choice, with or
        without a ``repetition_penalty``, is one ``ops.decode_select`` launch, token-identical to the eager loop.

        ``sampling=True`` also graphs ``use_nucleus_sampling`` (temperature + top-p).  Its draws come from the kernel's
        counter-based generator (Philox4x32-10 keyed by a per-call seed taken from the caller's ``generator``, by
        row and by step): a seeded call reproduces itself, but the tokens are NOT those of the eager loop, whose
        ``torch.multinomial`` consumes the generator differently.  Without it, sampled decoding runs eagerly.

        Beam search (``num_beams > 1``, within ``ops.beam_select_supported``: at most 8 beams and 4 eos ids) is graphed
        too: one replay per step of ``ops.beam_select`` + ``ops.kv_beam_reorder`` + the decoder, with the eager loop's
        tokens.  One caveat: the kernel's log-softmax sums in a different order from ``torch.log_softmax``, so graphed
        and eager tokens can differ where two candidates' scores are within a few fp32 ulps of each other.

        With ``sampling=True`` beam sample (``num_beams > 1`` with ``use_nucleus_sampling``, within
        ``ops.beam_sample_supported``) is graphed as well: ``ops.beam_sample`` + ``ops.kv_beam_reorder`` + the decoder,
        its draws from the kernel's Philox stream keyed by a per-call seed, so again not the eager loop's tokens."""
        self._decode_graphs = {} if enabled else None
        self._decode_graph_sampling = bool(enabled and sampling)
        return self

    def prepare(self, text_ids, visual_output, num_image_per_seq, max_num_image: int):
        st = self.special_token_dict
        embeds = self.mm_decoder.embed_tokens(text_ids)
        mm_embeds = splice_image_embeds(embeds, text_ids, visual_output["vis_embed"], self.soi_token,
                                        st["image_token_id"], st["soi_token_id"])
        cross = cross_attention_mask_from_ids(text_ids, max_num_image, st["bos_token_id"], st["soi_token_id"],
                                              num_image_per_seq)
        feats = pack_mmfs_features(visual_output["multiscale_features"], self.spatial_shapes, num_image_per_seq,
                                   max_num_image)
        return mm_embeds, cross, feats

    def forward(self, text_ids, visual_output, num_image_per_seq, max_num_image: int, attention_mask=None):
        mm_embeds, cross, feats = self.prepare(text_ids, visual_output, num_image_per_seq, max_num_image)
        out = self.mm_decoder(inputs_embeds=mm_embeds, attention_mask=attention_mask, vision_hidden_states=feats,
                              cross_attention_mask=cross, use_cache=False, return_dict=True)
        return self.text_decoder.logits(out.last_hidden_state)

    @torch.no_grad()
    def generate_images(self, text_ids, visual_output, num_image_per_seq, max_num_image: int, attention_mask=None,
                        target_image_idxs=None, **kwargs):
        """``MMInterleaved.generate_images`` (mm_interleaved.py:520-596): decoder prefill over the interleaved context,
        per-image reversed context features (:254-304) and previous-image MMFS features (:306-340), optional selection
        of target images, then ``ImageDecoder.generate_images`` (Q-Former -> CFG denoise loop with the MMFS network)."""
        if self.image_decoder is None:
            raise RuntimeError("generate_images needs an image_decoder (ImageDecoder with a UNet and an MMFSNet)")
        st = self.special_token_dict
        mm_embeds, cross, feats = self.prepare(text_ids, visual_output, num_image_per_seq, max_num_image)
        hidden = self.mm_decoder(inputs_embeds=mm_embeds, attention_mask=attention_mask, vision_hidden_states=feats,
                                 cross_attention_mask=cross, use_cache=False, return_dict=True).last_hidden_state
        ms = visual_output["multiscale_features"]
        n_img = ms[0].shape[0]
        mmfs_features, mmfs_mask = mmfs_features_for_image_decoder(ms, text_ids, st["soi_token_id"])
        ctx, ctx_mask = context_features_for_image_decoder(hidden, text_ids, st["soi_token_id"], self.context_feat_proj,
                                                           self.seq_len, n_img, pad_to=kwargs.pop("context_pad_to", None))
        if target_image_idxs is not None:
            ctx, ctx_mask, mmfs_mask = (torch.index_select(t, 0, target_image_idxs) for t in (ctx, ctx_mask, mmfs_mask))
            mmfs_features = [torch.index_select(f, 0, target_image_idxs) for f in mmfs_features]
        out = self.image_decoder.generate_images(context_features=ctx, context_attention_mask=ctx_mask,
                                                 mmfs_features=mmfs_features, mmfs_mask=mmfs_mask, **kwargs)
        out.update(context_features=ctx, context_attention_mask=ctx_mask, mmfs_mask=mmfs_mask)
        return out

    @torch.no_grad()
    def generate_texts(self, text_ids, visual_output, num_image_per_seq, max_num_image: int, attention_mask=None,
                       max_new_tokens: int = 30, eos_token_id=2, pad_token_id: int = 0, static_cache: bool = True,
                       min_length: int = 0, repetition_penalty: float = 1.0, use_nucleus_sampling: bool = False,
                       top_p: float = 0.9, temperature: float = 1.0, generator: Optional[torch.Generator] = None,
                       num_beams: int = 1, length_penalty: float = 1.0, num_return_sequences: int = 1):
        """Text continuation over the interleaved context -- ``MMInterleaved.generate_texts``
        (mm_interleaved.py:598-664), which drives HF ``generate`` through ``CascadeLlamaForCausalLMWrapper``
        (models/utils/causal_lm_cascade.py:91-204): prefill on ``inputs_embeds`` with the image features, then one
        token per step over the KV cache, the last row of the cross-attention mask serving every new token
        (mmfs.py:161-162), ``position_ids = cumsum(mask) - 1`` (causal_lm_cascade.py:179-185).  Batches are expected
        left-padded (collator.py:337).  Greedy by default (num_beams=1, do_sample=False: the release inference
        config); the reference's other knobs that do not need beams are honoured with HF's semantics:
        ``repetition_penalty`` (scores of already generated ids divided / multiplied), ``min_length`` (every eos id
        is suppressed while fewer than ``min_length`` tokens were generated), several ``eos_token_id`` values (the
        reference passes [eos, soi]), and ``use_nucleus_sampling`` = temperature + top-p sampling.  ``num_beams > 1``
        runs HF-style beam search (``generation.beam_search``; the reference's captioning default is 5 beams) and returns
        (B * num_return_sequences, <= max_new_tokens) padded ids; otherwise (B, max_new_tokens) ids.  ``num_beams > 1``
        with ``use_nucleus_sampling`` is HF 4.31's beam sample (the same loop: temperature, top-k 50 and top-p on
        the beam scores, 2 * num_beams candidates drawn per sequence, ``num_return_sequences`` independent searches
        per prompt); it raises ``ValueError`` where 4.31 does, when a step leaves fewer than num_beams non-eos
        candidates.

        Under ``enable_decode_graphs()`` greedy decoding (with or without the penalty, vocabularies up to
        ``ops.SELECT_MAX_V``) replays one CUDA graph per token with the eager loop's tokens; nucleus sampling is graphed only after ``enable_decode_graphs(True,
        sampling=True)``, and then draws from the kernel's Philox stream instead of ``torch.multinomial`` (same
        distribution, different tokens for a given ``generator`` seed).  Beam search replays one graph per step when
        its sizes are within ``ops.beam_select_supported`` (else it runs the eager loop), with the eager loop's tokens
        except where two candidates' scores lie within a few fp32 ulps (the kernel's log-softmax sums in another
        order than ``torch.log_softmax``).  Beam sample is graphed under ``enable_decode_graphs(True, sampling=True)``
        within ``ops.beam_sample_supported``, with Philox draws like graphed nucleus sampling."""
        return generation.generate_texts(self, text_ids, visual_output, num_image_per_seq, max_num_image, attention_mask,
                                         max_new_tokens, eos_token_id, pad_token_id, static_cache, min_length,
                                         repetition_penalty, use_nucleus_sampling, top_p, temperature, generator,
                                         num_beams, length_penalty, num_return_sequences)


def _llm_config_from(llm_config, llm_model_path, txt_vocab_size, image_embed_dim, cross_attention_frequency, spatial_shapes):
    """``LlamaConfig.from_pretrained(llm_model_path)`` + the three MMFS additions (mm_interleaved.py:59-69) without
    transformers: reads ``<llm_model_path>/config.json``.  Returns (LlamaMMFSConfig, original vocabulary size)."""
    import dataclasses
    import json
    import os
    if llm_config is None:
        cfg_file = os.path.join(str(llm_model_path), "config.json")
        if not os.path.exists(cfg_file):
            raise FileNotFoundError(f"{cfg_file} not found: pass llm_model_path (a directory holding the Llama config.json) "
                                    "or llm_config=LlamaMMFSConfig(...)")
        raw = json.load(open(cfg_file))
        names = {f.name for f in dataclasses.fields(LlamaMMFSConfig)}
        llm_config = LlamaMMFSConfig(**{k: v for k, v in raw.items() if k in names})
    elif isinstance(llm_config, dict):
        llm_config = LlamaMMFSConfig(**llm_config)
    else:
        llm_config = dataclasses.replace(llm_config)
    orig_vocab = llm_config.vocab_size if llm_config.vocab_size < txt_vocab_size else txt_vocab_size - 2
    llm_config.vocab_size = txt_vocab_size                     # resize_token_embeddings (:72)
    llm_config.image_embed_dim = image_embed_dim
    llm_config.cross_attention_frequency = cross_attention_frequency
    llm_config.spatial_shapes = list(spatial_shapes)
    return llm_config, orig_vocab


class MMInterleaved(InterleavedForward):
    """The reference's top-level model surface (mm_interleaved/models/mm_interleaved.py:25-763) on this repo's modules:
    same constructor keywords (:26-49), same sub-module / parameter names (``visual_tokenizer``, ``mm_decoder``,
    ``text_decoder``, ``image_decoder``, ``context_feat_proj``, ``soi_token``), and the same entry points
    ``forward(text_ids, image_tensors, ...)`` (:408-518), ``generate_texts`` (:598-664), ``generate_images`` (:520-596),
    ``generate_scores`` (:666-743) and ``generate(mode, **batch)`` (:745-763) -- so ``inference.py`` / ``evaluate.py``
    drive it with their unchanged batches (``model.generate(mode=..., **inputs)``, inference.py:237-269).

    Differences a caller can see: weights are not fetched by the constructor (``llm_model_path`` is only read for its
    ``config.json``; the reference's ``load_model_weights`` fills the parameters afterwards); ``forward`` computes the
    text loss (and returns the logits), and adds the image-decoder loss ``loss_img`` when the image decoder's VAE has
    an encoder (``image_decoder_config={"vae": {"with_encoder": True}}``) -- evaluation losses only, there is no
    backward; ``generate_images`` returns latents as ``image`` unless the image decoder has a VAE (``image_decoder_config``
    with ``vae=True`` builds the SD-2.1 decoder, vae_sd.py) or a ``vae_decode`` callable is attached to
    ``image_decoder.decoder``.  Extension keyword: ``llm_config`` (a ``LlamaMMFSConfig`` / dict) replaces
    ``llm_model_path``; ``max_num_image`` in a batch skips the one host sync on ``num_image_per_seq.max()``."""

    def __init__(self, *, llm_model_path="", seq_len=2048, txt_vocab_size=32002, loss_img_weight=10.0, loss_txt_weight=1.0,
                 special_token_dict: Optional[dict] = None, visual_tokenizer_config=None, image_decoder_config=None,
                 use_llama_gradient_checkpointing=True, num_img_token=64, image_embed_dim=1024, cross_attention_frequency=4,
                 spatial_shapes=(32, 16, 8), dataset_to_ignore_noimage_cond_loss=(), llm_config=None,
                 visual_tokenizer: Optional[nn.Module] = None, image_decoder: Optional[nn.Module] = None):
        cfg, orig_vocab = _llm_config_from(llm_config, llm_model_path, txt_vocab_size, image_embed_dim,
                                           cross_attention_frequency, spatial_shapes)
        if image_decoder is None and image_decoder_config is not None:
            image_decoder = ImageDecoder(**dict(image_decoder_config), mmfs_input_channel=image_embed_dim)
        super().__init__(cfg, special_tokens=special_token_dict, orig_vocab_size=orig_vocab, seq_len=seq_len,
                         image_decoder=image_decoder)
        if visual_tokenizer is None:            # (extension: a pre-built module may be passed instead of its config)
            from .visual_tokenizer import VisualTokenizer
            visual_tokenizer = VisualTokenizer(llm_hidden_size=cfg.hidden_size, **dict(visual_tokenizer_config or {}))
        self.visual_tokenizer = visual_tokenizer
        self.txt_vocab_size = txt_vocab_size
        self.loss_img_weight, self.loss_txt_weight = loss_img_weight, loss_txt_weight
        self.num_img_token = num_img_token
        self.dataset_to_ignore_noimage_cond_loss = list(dataset_to_ignore_noimage_cond_loss)
        self.mm_decoder.gradient_checkpointing = use_llama_gradient_checkpointing      # used under autograd only
        self._tok_graph = None

    # ---------------------------------------------------------------------------------------------------------
    def enable_cuda_graphs(self, tokenizer: bool = True) -> "MMInterleaved":
        """Replay the visual tokenizer (~2400 small kernels per 16 images) from a CUDA graph captured once per
        image-batch shape (SURVEY.md 8 f3).  Inference only; the tokenizer's outputs then live in static buffers that
        the next call overwrites -- everything this class returns to the caller is cloned out of them."""
        from ._graphs import GraphedCallable
        self._tok_graph = GraphedCallable(self.visual_tokenizer) if tokenizer else None
        sd = getattr(getattr(self, "image_decoder", None), "decoder", None)
        if sd is not None and hasattr(sd, "enable_cuda_graphs"):
            sd.enable_cuda_graphs(True)                  # UNet evaluation graph, kept across generate_images calls
        return self

    def _tokenize(self, image_tensors):
        p = self.visual_tokenizer.proj.weight
        image_tensors = image_tensors.to(device=p.device, dtype=p.dtype)
        if self._tok_graph is not None and image_tensors.is_cuda and not torch.is_grad_enabled():
            out = self._tok_graph(image_tensors)
            return dict(out, _static=True)
        return self.visual_tokenizer(image_tensors)

    @staticmethod
    def _owned(visual_output):
        """The multi-scale maps as tensors the caller may keep (cloned when they alias CUDA-graph buffers)."""
        ms = visual_output["multiscale_features"]
        return [f.clone() for f in ms] if visual_output.get("_static") else ms

    # ---------------------------------------------------------------------------------------------------------
    def _max_num_image(self, num_image_per_seq, max_num_image=None):
        return int(max_num_image) if max_num_image is not None else int(num_image_per_seq.max())   # :194

    def _prepare_mm_embeds(self, text_ids, image_tensors=None, num_image_per_seq=None, meta=None, max_num_image=None):
        """mm_interleaved.py:121-183: tokenizer on the images, embed splice, visibility mask, MMFS feature packing."""
        num_image_per_seq = num_image_per_seq.reshape(-1).to(text_ids.device)
        visual_output = self._tokenize(image_tensors)
        mm_embeds, cross, feats = self.prepare(text_ids, visual_output, num_image_per_seq,
                                               self._max_num_image(num_image_per_seq, max_num_image))
        return {"mm_embeds": mm_embeds, "cross_attention_mask": cross, "mmfs_features_mm": feats,
                "multiscale_features": self._owned(visual_output), "_visual_output": visual_output}

    def _prepare_gt_text_ids(self, text_ids, attention_mask=None, ignore_prompt_token_offset=0, gt_text_ids=None, meta=None):
        """mm_interleaved.py:342-406 (next-token targets with prompt / pad / image / bos positions set to -100)."""
        st = self.special_token_dict
        if gt_text_ids is not None:
            return gt_text_ids[..., 1:]
        gt = text_ids.clone()
        if isinstance(ignore_prompt_token_offset, int):
            gt[:, :ignore_prompt_token_offset] = -100
        else:
            assert len(ignore_prompt_token_offset) == gt.shape[0]
            for idx, offset in enumerate(ignore_prompt_token_offset):
                gt[idx, :offset] = -100
        if meta is not None and meta.get("dataset_name") in self.dataset_to_ignore_noimage_cond_loss:
            pos = torch.arange(text_ids.shape[-1], device=text_ids.device)[None, :].expand_as(text_ids)
            nearest_bos = pos.masked_fill(text_ids != st["bos_token_id"], -1).cummax(dim=1).values.clamp(min=0)
            nearest_soi = pos.masked_fill(text_ids != st["soi_token_id"], -1).cummax(dim=1).values
            gt = gt.masked_fill((nearest_soi < nearest_bos) | (nearest_soi == -1), -100)
        gt = gt[:, 1:]
        nxt = text_ids[:, 1:]
        gt = gt.masked_fill(nxt == st["pad_token_id"], -100).masked_fill(nxt == st["image_token_id"], -100)
        if attention_mask is not None:
            gt = gt.masked_fill(attention_mask[:, 1:] == 0, -100)
        bos2soi = (text_ids[:, :-1] == st["bos_token_id"]) & (nxt == st["soi_token_id"])
        return gt.masked_fill(bos2soi, -100).masked_fill(nxt == st["bos_token_id"], -100)

    def forward(self, text_ids, image_tensors=None, image_tensors_dec=None, num_image_per_seq=None, attention_mask=None,
                gt_text_ids=None, nearest_bos_idxs=None, ignore_prompt_token_offset=0, loss_img_weight=None,
                loss_txt_weight=None, meta=None, image_loss_mask=None, **kwargs):
        """mm_interleaved.py:408-518.  Returns ``loss_txt`` / ``loss`` like the reference plus ``text_logits`` (B, T, V)
        (extension; ``return_loss=False`` stops there -- the "step" of SURVEY.md 8d).  When the image decoder's VAE has
        an encoder, the image loss is added as in the reference: ``ImageDecoder.forward`` on ``image_tensors_dec`` (else
        ``image_tensors``) with the per-image contexts and previous-image MMFS features (from ``nearest_bos_idxs``),
        ``loss_img`` = its detached mean and ``loss = loss_txt * w_txt + loss_img * w_img``; ``multiscale_features``
        then leaves the output, as there.  ``generator`` (keyword) seeds the image loss's random draws.
        Under autograd the text loss is differentiable (``freeze_like_reference``), down to the visual tokenizer's head
        (``pos_proj``, ``pos_ln``, ``post_ln``, the Q-Former, ``proj``) and its ViT-Adapter, through the frozen CLIP ViT
        (``visual_tokenizer.freeze_like_reference()``).  The image loss is differentiable too, through the frozen SD UNet
        (``image_decoder.decoder.unet.requires_grad_(False)``): its gradient reaches the image decoder's Q-Former,
        ``neg_prompt_embeds``, the MMFS hook, ``context_feat_proj`` and, through the context and the MMFS features, the
        LLM and the visual tokenizer.  A trainable CLIP ViT weight or, with the image loss on, a trainable UNet weight
        raises up front, as neither has a backward here."""
        if records(self):
            if any(p.requires_grad for n, p in self.visual_tokenizer.encoder.vision_model.named_parameters()
                   if not n.startswith("adapter")):
                raise RuntimeError("MMInterleaved.forward under autograd: the visual tokenizer has no backward here "
                                   "for its CLIP ViT weights (the reference freezes them, and trains the ViT-Adapter); "
                                   "call model.visual_tokenizer.freeze_like_reference(), or freeze the whole encoder "
                                   "(model.visual_tokenizer.encoder.requires_grad_(False)), or run under torch.no_grad()")
            if self._has_image_loss() and not self._image_loss_differentiable():
                raise RuntimeError("MMInterleaved.forward under autograd: the image-decoder loss has no backward here "
                                   "for the UNet's own weights (it trains what feeds the UNet); freeze them with "
                                   "model.image_decoder.decoder.unet.requires_grad_(False), or build the image decoder's "
                                   "VAE without an encoder (no image loss), or run under torch.no_grad()")
        return_loss = kwargs.pop("return_loss", True)
        generator = kwargs.pop("generator", None)
        out = self._prepare_mm_embeds(text_ids, image_tensors, num_image_per_seq, meta, kwargs.pop("max_num_image", None))
        mm = self.mm_decoder(inputs_embeds=out.pop("mm_embeds"), attention_mask=attention_mask,
                             vision_hidden_states=out.pop("mmfs_features_mm"),
                             cross_attention_mask=out.pop("cross_attention_mask"), use_cache=False, return_dict=True)
        out.pop("_visual_output")
        logits = self.text_decoder.logits(mm.last_hidden_state)
        if not return_loss:
            out["text_logits"] = logits
            return out
        gt = self._prepare_gt_text_ids(text_ids, attention_mask, ignore_prompt_token_offset, gt_text_ids, meta)
        loss_txt = F.cross_entropy(logits[:, :-1].float().transpose(1, 2), gt.contiguous(), reduction="mean")   # :458-463
        w = self.loss_txt_weight if loss_txt_weight is None else loss_txt_weight
        out.update(loss_txt=loss_txt.detach(), loss=loss_txt * w, text_logits=logits)
        if self._has_image_loss():                                                                    # :478-515
            st = self.special_token_dict
            ms = out.pop("multiscale_features")
            ctx, ctx_mask = context_features_for_image_decoder(mm.last_hidden_state, text_ids, st["soi_token_id"],
                                                               self.context_feat_proj, self.seq_len, ms[0].shape[0],
                                                               nearest_bos_idxs=nearest_bos_idxs)
            mmfs_features, mmfs_mask = mmfs_features_for_image_decoder(ms, text_ids, st["soi_token_id"], nearest_bos_idxs)
            loss_img = self.image_decoder(image_tensors=image_tensors if image_tensors_dec is None else image_tensors_dec,
                                          context_features=ctx, context_attention_mask=ctx_mask,
                                          image_loss_mask=image_loss_mask, mmfs_features=mmfs_features,
                                          mmfs_mask=mmfs_mask, generator=generator).mean()
            wi = self.loss_img_weight if loss_img_weight is None else loss_img_weight
            out.update(loss_img=loss_img.detach(), loss=out["loss"] + loss_img * wi)
        return out

    def freeze_like_reference(self):
        """The trainable set of the reference's constructor that this repository can differentiate (mm_interleaved.py:74-78,
        decoder_text.py:50-51): the LLM frozen except its ``llama_cross_attn`` blocks, the text head frozen except
        ``head_new``, ``soi_token`` trainable.  Returns ``self``.

        The reference also trains the visual tokenizer's ViT-Adapter and Q-Former head and the image decoder.  This
        leaves the tokenizer's flags as they are.  Its head (``pos_proj``, ``pos_ln``, ``post_ln``, the Q-Former,
        ``proj``) and its ViT-Adapter have a backward here, its CLIP ViT weights do not: ``forward`` under autograd
        raises while a CLIP ViT parameter requires grad, or while the image loss is on and a UNet parameter requires
        grad.  The image decoder's flags are left as they are too: its Q-Former, ``neg_prompt_embeds`` and MMFS hook
        have a backward, the UNet's own weights do not (``model.image_decoder.decoder.unet.requires_grad_(False)``).
        To train the text loss like the reference, call ``model.freeze_like_reference();
        model.visual_tokenizer.freeze_like_reference()``; to keep the adapter frozen, freeze the encoder
        (``model.visual_tokenizer.encoder.requires_grad_(False)``); to train without the tokenizer, freeze all of it
        (``model.visual_tokenizer.requires_grad_(False)``)."""
        for name, p in self.mm_decoder.named_parameters():
            p.requires_grad_("llama_cross_attn" in name)
        self.text_decoder.requires_grad_(False)
        self.text_decoder.head_new.requires_grad_(True)
        self.soi_token.requires_grad_(True)
        return self

    def _has_image_loss(self) -> bool:
        sd = getattr(self.image_decoder, "decoder", None)
        return getattr(getattr(sd, "vae", None), "encoder", None) is not None

    def _image_loss_differentiable(self) -> bool:
        """The image loss has a backward when the image decoder runs this repository's UNet with its weights frozen."""
        from .unet_sd import UNet2DConditionModel, has_trainable_weights
        unet = getattr(getattr(self.image_decoder, "decoder", None), "unet", None)
        return isinstance(unet, UNet2DConditionModel) and not has_trainable_weights(unet)

    @torch.no_grad()
    def generate_texts(self, text_ids, image_tensors=None, num_image_per_seq=None, attention_mask=None, meta=None, **kwargs):
        """mm_interleaved.py:598-664 with its BLIP-2 defaults (max_length 30, min_length 8, 5 beams, eos = [eos, soi])."""
        st = self.special_token_dict
        num_captions = kwargs.pop("num_captions", 1)
        max_length = kwargs.pop("max_length", 30)
        min_length = kwargs.pop("min_length", 8)
        num_beams = kwargs.pop("num_beams", 5)
        nucleus = kwargs.pop("use_nucleus_sampling", False)
        top_p = kwargs.pop("top_p", 0.9)
        repetition_penalty = kwargs.pop("repetition_penalty", 1.0)
        length_penalty = kwargs.pop("length_penalty", 1.0)
        temperature = kwargs.pop("temperature", 1)
        num_image_per_seq = num_image_per_seq.reshape(-1).to(text_ids.device)
        visual_output = self._tokenize(image_tensors)
        ids = super().generate_texts(text_ids, visual_output, num_image_per_seq,
                                     self._max_num_image(num_image_per_seq, kwargs.pop("max_num_image", None)),
                                     attention_mask=attention_mask, max_new_tokens=max_length,
                                     eos_token_id=[st.get("eos_token_id", 2), st["soi_token_id"]],
                                     pad_token_id=st.get("pad_token_id", 0), min_length=min_length,
                                     repetition_penalty=repetition_penalty, use_nucleus_sampling=nucleus, top_p=top_p,
                                     temperature=temperature, generator=kwargs.pop("generator", None), num_beams=num_beams,
                                     length_penalty=length_penalty, num_return_sequences=num_captions)
        return {"multiscale_features": self._owned(visual_output), "text_ids": ids}

    @torch.no_grad()
    def generate_images(self, text_ids, image_tensors=None, num_image_per_seq=None, attention_mask=None, meta=None,
                        target_image_idxs=None, **kwargs):
        """mm_interleaved.py:520-596."""
        num_image_per_seq = num_image_per_seq.reshape(-1).to(text_ids.device)
        visual_output = self._tokenize(image_tensors)
        return super().generate_images(text_ids, visual_output, num_image_per_seq,
                                       self._max_num_image(num_image_per_seq, kwargs.pop("max_num_image", None)),
                                       attention_mask=attention_mask, target_image_idxs=target_image_idxs, **kwargs)

    @torch.no_grad()
    def generate_scores(self, text_ids, image_tensors=None, num_image_per_seq=None, attention_mask=None, options_ids=None,
                        options_attn_masks=None, **kwargs):
        """mm_interleaved.py:666-743: for sample i, the log-likelihood of every answer option appended to its context,
        summed over the option's unmasked tokens; mini-batches of 4 options.  The image of a sample is tokenised ONCE and
        its outputs are expanded over the options (the reference re-encodes the same image per option row)."""
        import math
        scores = []
        for i in range(len(text_ids)):
            n_opt = options_ids[i].shape[0]
            offset = len(text_ids[i])
            ids = torch.cat((text_ids[i][None].expand(n_opt, -1), options_ids[i]), dim=1)
            mask = torch.cat((attention_mask[i][None].expand(n_opt, -1), options_attn_masks[i]), dim=1)
            vis1 = self._tokenize(image_tensors[[i]])
            n_i = num_image_per_seq[[i]].reshape(-1).to(ids.device)
            if int(n_i.numel()) != 1 or image_tensors[[i]].shape[0] != 1:
                raise RuntimeError("generate_scores expects one image per sample (mm_interleaved.py:684-689)")
            mini_bs = 4
            chunks = []
            for j in range(math.ceil(n_opt / mini_bs)):
                sl = slice(j * mini_bs, (j + 1) * mini_bs)
                nb = ids[sl].shape[0]
                vis = {"vis_embed": vis1["vis_embed"].expand(nb, -1, -1),
                       "multiscale_features": [f.expand(nb, -1, -1, -1) for f in vis1["multiscale_features"]]}
                mm_embeds, cross, feats = self.prepare(ids[sl], vis, n_i.expand(nb), 1)
                hid = self.mm_decoder(inputs_embeds=mm_embeds, attention_mask=mask[sl], vision_hidden_states=feats,
                                      cross_attention_mask=cross, use_cache=False, return_dict=True).last_hidden_state
                chunks.append(self.text_decoder.logits(hid[:, offset - 1:-1]))
            logits = torch.cat(chunks)
            assert logits.shape[1] == options_ids[i].shape[1]
            logp = F.log_softmax(logits.float(), dim=-1).gather(-1, options_ids[i][..., None]).squeeze(-1)
            scores.append((logp * options_attn_masks[i]).sum(dim=-1))
        return {"scores": torch.stack(scores, dim=0)[:, None, :]}

    @torch.no_grad()
    def generate_interleaved(self, text_ids, image_tensors, num_image_per_seq, attention_mask=None,
                             generate_mode="generate_texts", num_iter=2, auto_end=False, force_gen_image_next=False,
                             force_replace_gen_text=False, generator: Optional[torch.Generator] = None, **kwargs):
        """Interleaved image-text generation of ONE sample (batch 1) in one call: the turn loop of the reference's
        ``inference.py::inference_all`` (text turns as ``generate_texts``, image turns as ``generate_images``,
        ``update_texts`` / ``update_image`` between them, ``auto_end``, ``force_gen_image_next``) on an
        ``interleaved.InterleavedSession`` that keeps the KV cache, the hidden states and the tokenizer outputs across
        turns, so every position is prefilled once and every image tokenized once, and re-enters each generated image
        on the device (``ops.image_reentry``).  ``kwargs``: the generation keywords of ``mm_inference.yaml``
        (``max_length``, ``min_length``, ``num_beams``, ``use_nucleus_sampling``, ``top_p``, ``temperature``,
        ``repetition_penalty``, ``length_penalty``, ``guidance_scale``, ``num_inference_steps``,
        ``num_validation_images``), ``max_cache_length`` (refuse samples that could outgrow it) and ``return_session``.
        Needs an image decoder with a VAE decoder; ``force_replace_gen_text`` (a text tokenizer's job) raises.
        Returns ``turns`` and the final ``text_ids``, ``attention_mask``, ``image_tensors``, ``num_image_per_seq``."""
        from .interleaved import generate_interleaved
        return generate_interleaved(self, text_ids, image_tensors, num_image_per_seq, attention_mask, generate_mode,
                                    num_iter, auto_end, force_gen_image_next, force_replace_gen_text, generator, **kwargs)

    def generate(self, mode="generate_images", **kwargs):
        """mm_interleaved.py:745-763."""
        if mode in ("generate_images", "generate_segm"):
            assert self.image_decoder is not None
            return self.generate_images(**kwargs)
        if mode in ("generate_texts", "generate_vqa", "generate_grounding"):
            assert self.text_decoder is not None
            return self.generate_texts(**kwargs)
        if mode == "generate_scores":
            assert self.text_decoder is not None
            return self.generate_scores(**kwargs)
        raise NotImplementedError
