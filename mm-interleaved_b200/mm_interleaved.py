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

from ._cache import WeightCache
from .llama_mmfs import LlamaMMFSConfig, LlamaModel

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
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
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
        scaling factor.  The VAE encodes in its own dtype (the reference casts it to fp32)."""
        n = self.vae_encode_mini_bs if self.vae_encode_mini_bs > 0 else image.shape[0]
        parts = [self.vae.encode(image[i:i + n]).latent_dist.sample(generator).to(dtype) for i in range(0, image.shape[0], n)]
        return torch.cat(parts, dim=0) * self.vae_scaling_factor

    def forward(self, image, text_embeds, return_outputs=False, mmfs_features=None, mmfs_mask=None,
                generator: Optional[torch.Generator] = None):
        """The denoising loss of sd.py:240-316 (inference kernels: an evaluation loss, call under ``torch.no_grad()``).
        ``image`` (B, 3, S, S) in [0, 1] with S = ``image_size``; returns the per-element
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
        ``image_loss_mask`` is 0, then averaged over every element, zeroed ones included."""
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


class _GraphedDecoder:
    """Static state + one CUDA graph of a decode step for ``InterleavedForward`` (see ``enable_decode_graphs``).

    Everything that changes from token to token lives in DEVICE tensors the graph updates itself -- the slot the new
    key/value row goes to, the key mask over the whole static cache, the position ids, the step counter, the finished
    flags, the output ids -- so generating N tokens is N ``graph.replay()`` calls with no host synchronisation.  The
    image-side tensors of the cross-attention layers are a ``PreparedVision`` over static storage, refilled eagerly once
    per call (a graph replay bypasses Python, so nothing inside the graph may depend on a tensor-identity cache).

    ``mode``: None = plain greedy (processors + arg-max in torch ops); ``"greedy"`` (with a repetition penalty) and
    ``"sample"`` (temperature + top-p) choose the token with ``ops.decode_select``, which reads the penalty,
    temperature, top_p and seed from device buffers written once per call, so one graph serves any of their values.
    ``"beam"``: beam search over B * num_beams rows (``generate_beams``); the step is ``ops.beam_select`` (scores,
    hypotheses, done flags, history) -> ``ops.kv_beam_reorder`` (the generated positions of every layer's K and V, held
    in one tensor ``kv``) -> the decoder on the next tokens, with the repetition and length penalties in a device
    buffer.  ``finished`` then holds the per-sequence done flags.  ``"beam_sample"``: the same with ``ops.beam_sample``
    (temperature and top_p in the device buffer too, one seed per call as ``"sample"``, a sticky error flag) and every
    beam starting at score 0."""

    def __init__(self, owner, B, t_max, feats_shape, dtype, device, eos_ids, pad_id, min_length, max_new, mode=None,
                 num_beams=1):
        from . import ops
        from .llama_mmfs import PreparedVision, StaticKV
        self.owner, self.B, self.t_max, self.max_new, self.min_length = owner, B, t_max, max_new, int(min_length)
        self.mode, self.pad_id, self.nb = mode, int(pad_id), int(num_beams)
        R = B * self.nb                                                     # decoder rows: one per beam
        model = owner.mm_decoder
        n_img = feats_shape[1]
        if mode in ("beam", "beam_sample"):
            H = model.config.num_attention_heads
            self.kv = torch.zeros((2 * len(model.layers), R, t_max, H, model.config.hidden_size // H), dtype=dtype,
                                  device=device)
            self.past = [StaticKV.over(self.kv[2 * i], self.kv[2 * i + 1]) for i in range(len(model.layers))]
        else:
            self.past = model.static_cache(B, t_max, dtype=dtype, device=device)
        self.pv = PreparedVision((R,) + tuple(feats_shape[1:]))
        probe = model.prepare_vision(torch.zeros(feats_shape, dtype=dtype, device=device))
        for idx, val in probe.values.items():
            self.pv.values[idx] = val.new_empty((R,) + tuple(val.shape[1:]))
        V = owner.text_decoder.head.weight.shape[0]
        self.logits = torch.zeros((R, V), dtype=torch.float32, device=device)
        self.key_mask = torch.zeros((R, t_max), dtype=torch.uint8, device=device)
        self.pos = torch.zeros((R, 1), dtype=torch.long, device=device)
        self.cur = torch.zeros((1,), dtype=torch.long, device=device)
        self.step = torch.zeros((1,), dtype=torch.long, device=device)
        self.finished = torch.zeros((B,), dtype=torch.bool, device=device)
        self.out_ids = torch.zeros((B, max_new), dtype=torch.long, device=device)
        self.cross_last = torch.zeros((R, 1, n_img), dtype=torch.float32, device=device)
        self.eos = torch.tensor(eos_ids, dtype=torch.long, device=device) if eos_ids else None
        self.pad = torch.tensor(int(pad_id), dtype=torch.long, device=device)
        self.neg_inf = torch.tensor(float("-inf"), dtype=torch.float32, device=device)
        self.zero = torch.zeros((), dtype=torch.float32, device=device)
        if mode is not None:
            self.next_ids = torch.zeros((R, 1), dtype=torch.long, device=device)
        if mode in ("greedy", "sample"):
            self.params = torch.ones((3,), dtype=torch.float32, device=device)   # penalty, temperature, top_p
            self.seed = torch.zeros((1,), dtype=torch.long, device=device)
        if mode in ("beam", "beam_sample"):
            nb = self.nb
            # repetition_penalty, length_penalty (+ temperature, top_p when sampling)
            self.params = torch.ones((2 if mode == "beam" else 4,), dtype=torch.float64, device=device)
            self.beam_scores = torch.zeros((R,), dtype=torch.float32, device=device)
            self.history = torch.zeros((R, max_new), dtype=torch.long, device=device)
            self.parent = torch.zeros((R,), dtype=torch.long, device=device)
            self.hyp_scores = torch.zeros((B, nb), dtype=torch.float64, device=device)
            self.hyp_ids = torch.zeros((B, nb, max_new), dtype=torch.long, device=device)
            self.hyp_meta = torch.zeros((B, nb, 2), dtype=torch.long, device=device)          # length (-1: free), serial
            n_scratch = R * ops.beam_candidates(nb, len(eos_ids)) if mode == "beam" else ops.beam_sample_scratch(nb, R)
            self.scratch = torch.zeros((n_scratch,), dtype=torch.long, device=device)
            self.all_done = torch.zeros((1,), dtype=torch.bool).pin_memory()                 # written by every replay
        if mode == "beam_sample":
            self.seed = torch.zeros((1,), dtype=torch.long, device=device)
            self.error = torch.zeros((1,), dtype=torch.int32, device=device)
        self.graph = None
        self.launches = 0
        self.replays = 0

    def _set_graph_mode(self, on: bool, length: int = 0):
        for c in self.past:
            c.slot = self.cur if on else None
            c.length = self.t_max - 1 if on else length

    def _step(self):
        """One token: processors + arg-max / draw on the pending logits, bookkeeping, decoder forward on the chosen token."""
        from . import ops
        o = self.owner
        if self.mode is None:
            scores = self.logits
            if self.eos is not None and self.min_length > 0:               # HF MinLengthLogitsProcessor
                bias = torch.where(self.step < self.min_length, self.neg_inf, self.zero)
                scores = scores.index_add(1, self.eos, bias.expand(self.B, self.eos.numel()).contiguous())
            nxt = scores.argmax(-1)
            if self.eos is not None:
                nxt = torch.where(self.finished, self.pad, nxt)
                self.finished.logical_or_((nxt[:, None] == self.eos[None, :]).any(dim=1))
            self.out_ids.index_copy_(1, self.step, nxt[:, None])
            fed = nxt[:, None]
        elif self.mode in ("beam", "beam_sample"):                         # scorer, then the cache follows the parents
            if self.mode == "beam":
                ops.beam_select(self.logits, self.step, self.params, self.beam_scores, self.history, self.next_ids,
                                self.parent, self.finished, self.hyp_scores, self.hyp_ids, self.hyp_meta, self.scratch,
                                self.nb, eos=self.eos, pad_id=self.pad_id, min_length=self.min_length)
            else:
                ops.beam_sample(self.logits, self.step, self.params, self.beam_scores, self.history, self.next_ids,
                                self.parent, self.finished, self.hyp_scores, self.hyp_ids, self.hyp_meta, self.error,
                                self.scratch, self.nb, eos=self.eos, pad_id=self.pad_id, min_length=self.min_length,
                                top_k=_BEAM_SAMPLE_TOP_K, seed=self.seed)
            ops.kv_beam_reorder(self.kv, self.parent, self.cur, self.step, self.nb, self.max_new, done=self.finished)
            fed = self.next_ids
        else:                                                              # processors, choice and bookkeeping: one kernel
            ops.decode_select(self.logits, self.out_ids, self.step, self.finished, self.next_ids, self.params, eos=self.eos,
                              pad_id=self.pad_id, min_length=self.min_length, sample=self.mode == "sample", seed=self.seed)
            fed = self.next_ids
        self.key_mask.index_fill_(1, self.cur, 1)                          # the fed token's cache slot becomes visible
        self.pos.add_(1)
        hid = o.mm_decoder(inputs_embeds=o.mm_decoder.embed_tokens(fed), attention_mask=self.key_mask,
                           position_ids=self.pos, past_key_values=self.past, vision_hidden_states=self.pv,
                           cross_attention_mask=self.cross_last, use_cache=True, return_dict=True).last_hidden_state
        self.logits.copy_(o.text_decoder.logits(hid)[:, -1].float())
        self.step.add_(1)
        self.cur.add_(1)
        if self.mode in ("beam", "beam_sample"):                           # read by the host two replays later
            self.all_done.copy_(self.finished.all().view(1), non_blocking=True)

    def _reset(self, L, attention_mask, position_ids, cross, logits0):
        self.key_mask.zero_()
        self.key_mask[:, :L].copy_(attention_mask.to(torch.uint8))
        self.pos.copy_(position_ids[:, -1:])
        self.cur.fill_(L)
        self.step.zero_()
        self.finished.zero_()
        self.out_ids.fill_(int(self.pad))
        self.cross_last.copy_(cross[:, -1:, :])
        self.logits.copy_(logits0)
        if self.mode == "beam":
            self.beam_scores.fill_(-1e9)
            self.beam_scores[::self.nb] = 0.0                              # only the first beam of a sequence is live
        if self.mode == "beam_sample":
            self.beam_scores.zero_()                                       # beam_sample starts every beam at 0
            self.error.zero_()
        if self.mode in ("beam", "beam_sample"):
            self.history.fill_(self.pad_id)
            self.hyp_scores.zero_()
            self.hyp_meta.fill_(-1)

    def _prefill_done(self, L, reset):
        """After the prefill: zero the unused cache slots, capture the step graph once, reset the per-call state."""
        from . import ops
        o = self.owner
        for c in self.past:                                                 # masked slots must hold finite numbers
            c.k[:, L:].zero_()
            c.v[:, L:].zero_()
        self._set_graph_mode(True)
        if self.graph is None:
            reset()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):                                          # lazy handles, weight-derived caches, RoPE tables
                    reset()                                                 # every warm-up step is step 0
                    self._step()
            torch.cuda.current_stream().wait_stream(side)
            reset()
            before = ops.launch_counter[0]
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._step()
            self.launches = ops.launch_counter[0] - before
            # the graph reads the RoPE tables by address: keep the captured storage alive even if an eager decode grows
            # (and so replaces) the shared tables later
            self._captured_rope = [l.self_attn._rope for l in o.mm_decoder.layers]
            for c in self.past:                                             # the warm-up steps wrote slots L, L+1
                c.k[:, L:].zero_()
                c.v[:, L:].zero_()
        reset()

    def generate(self, mm_embeds, cross, feats, attention_mask, position_ids, repetition_penalty=1.0, temperature=1.0,
                 top_p=1.0, generator=None):
        from . import ops
        o = self.owner
        B, L, _ = mm_embeds.shape
        if L + self.max_new > self.t_max:
            raise RuntimeError("prompt + new tokens exceed the captured cache length")
        if self.mode is not None:                                           # per-call values the graph reads on the device
            self.params[0].fill_(float(repetition_penalty))
            self.params[1].fill_(float(temperature))
            self.params[2].fill_(float(top_p))
            if self.mode == "sample":                                       # one seed per call, drawn on the device
                self.seed.random_(generator=generator)
        o.mm_decoder.prepare_vision(feats, out=self.pv)                     # eager, into the static buffers the graph reads
        self._set_graph_mode(False, 0)
        out = o.mm_decoder(inputs_embeds=mm_embeds, attention_mask=attention_mask, position_ids=position_ids,
                           past_key_values=self.past, vision_hidden_states=self.pv, cross_attention_mask=cross,
                           use_cache=True, return_dict=True)               # prefill straight into the static cache
        logits0 = o.text_decoder.logits(out.last_hidden_state[:, -1:])[:, -1].float()
        self._prefill_done(L, lambda: self._reset(L, attention_mask, position_ids, cross, logits0))
        for _ in range(self.max_new):
            self.graph.replay()
        ops.launch_counter[0] += self.launches * self.max_new
        self._set_graph_mode(False, L)
        return self.out_ids.clone()

    def generate_beams(self, mm_embeds, cross, feats, attention_mask, position_ids, repetition_penalty=1.0,
                       length_penalty=1.0, temperature=1.0, top_p=1.0, generator=None):
        """Beam search (``mode == "beam"`` or ``"beam_sample"``): the prompt is prefilled once per sequence and its
        cache rows, the ``PreparedVision`` values, key mask, position ids and last cross-attention row are replicated
        to the beams (beam sample: to the ``self.B // B`` independent searches of each prompt, then to their beams);
        then one replay per step.  At most two replays are in flight: before enqueuing replay t the host waits for
        replay t - 2 and reads the "all sequences done" flag it copied to pinned memory, so decoding stops at most two
        steps after the eager loop would (done sequences are inert).  Returns the host copies of the final state."""
        from . import ops
        o = self.owner
        B, L, _ = mm_embeds.shape
        if L + self.max_new > self.t_max:
            raise RuntimeError("prompt + new tokens exceed the captured cache length")
        self.params[0].fill_(float(repetition_penalty))
        self.params[1].fill_(float(length_penalty))
        if self.mode == "beam_sample":
            self.params[2].fill_(float(temperature))
            self.params[3].fill_(float(top_p))
            self.seed.random_(generator=generator)                          # one seed per call, drawn on the device
        rep = torch.arange(B, device=mm_embeds.device).repeat_interleave(self.B // B * self.nb)   # beam row -> prompt
        pv = o.mm_decoder.prepare_vision(feats)                             # the prefill's B rows, then one per beam
        for idx, val in pv.values.items():
            torch.index_select(val, 0, rep, out=self.pv.values[idx])
        pre = o.mm_decoder.static_cache(B, L, dtype=mm_embeds.dtype, device=mm_embeds.device)
        out = o.mm_decoder(inputs_embeds=mm_embeds, attention_mask=attention_mask, position_ids=position_ids,
                           past_key_values=pre, vision_hidden_states=pv, cross_attention_mask=cross, use_cache=True,
                           return_dict=True)
        logits0 = o.text_decoder.logits(out.last_hidden_state[:, -1:])[:, -1].float().index_select(0, rep)
        for dst, src in zip(self.past, pre):                                # a copy of the prompt rows, no recompute
            dst.k[:, :L].copy_(src.k.index_select(0, rep))
            dst.v[:, :L].copy_(src.v.index_select(0, rep))
        del pre, pv
        mask_r, pos_r, cross_r = (t.index_select(0, rep) for t in (attention_mask, position_ids, cross[:, -1:, :]))
        self._prefill_done(L, lambda: self._reset(L, mask_r, pos_r, cross_r, logits0))
        torch.cuda.current_stream().synchronize()                           # no copy into all_done is pending
        self.all_done.zero_()
        events = (torch.cuda.Event(), torch.cuda.Event())
        n = 0
        for t in range(self.max_new):
            if t >= 2:
                events[t % 2].synchronize()                                 # replay t - 2 has finished
                if bool(self.all_done[0]):
                    break
            self.graph.replay()
            events[t % 2].record()
            n += 1
        self.replays = n
        ops.launch_counter[0] += self.launches * n
        self._set_graph_mode(False, L)
        out = dict(history=self.history[:, :n].cpu(), beam_scores=self.beam_scores.cpu(), done=self.finished.cpu(),
                   hyp_scores=self.hyp_scores.cpu(), hyp_ids=self.hyp_ids.cpu(), hyp_meta=self.hyp_meta.cpu())
        if self.mode == "beam_sample":
            out["error"] = bool(self.error.item())
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
        later calls (SURVEY.md 8 f3; causal_lm_cascade.py:171-204 is the loop it replaces).  Greedy decoding with a
        ``repetition_penalty`` is graphed too (``ops.decode_select``), token-identical to the eager loop.

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

    def _decode_graph(self, mm_embeds, feats, max_new_tokens, eos_ids, pad_id, min_length, mode, num_beams=1, expand=1):
        """The ``_GraphedDecoder`` for this shape and these settings, built on first use (at most four are kept);
        ``expand`` independent beam searches per prompt (beam sample's ``num_return_sequences``)."""
        B, L, _ = mm_embeds.shape
        B *= expand
        t_max = ((L + max_new_tokens + 255) // 256) * 256                  # cache-length bucket: one graph serves nearby prompts
        key = (B, t_max, tuple(feats.shape), mm_embeds.dtype, mm_embeds.device, tuple(eos_ids), int(pad_id), int(min_length),
               int(max_new_tokens), int(num_beams), mode)
        dec = self._decode_graphs.get(key)
        if dec is None:
            if len(self._decode_graphs) >= 4:
                self._decode_graphs.pop(next(iter(self._decode_graphs)))
            dec = self._decode_graphs[key] = _GraphedDecoder(self, B, t_max, feats.shape, mm_embeds.dtype, mm_embeds.device,
                                                             eos_ids, pad_id, min_length, max_new_tokens, mode, num_beams)
        return dec

    @torch.no_grad()
    def _graphed_decode(self, mm_embeds, cross, feats, attention_mask, position_ids, max_new_tokens, eos_ids, pad_id,
                        min_length, mode, repetition_penalty, temperature, top_p, generator):
        dec = self._decode_graph(mm_embeds, feats, max_new_tokens, eos_ids, pad_id, min_length, mode)
        return dec.generate(mm_embeds, cross, feats, attention_mask, position_ids, repetition_penalty, temperature, top_p,
                            generator)

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
        runs HF-style beam search (``_beam_search`` below; the reference's captioning default is 5 beams) and returns
        (B * num_return_sequences, <= max_new_tokens) padded ids; otherwise (B, max_new_tokens) ids.  ``num_beams > 1``
        with ``use_nucleus_sampling`` is HF 4.31's beam sample (``_beam_sample``: temperature, top-k 50 and top-p on
        the beam scores, 2 * num_beams candidates drawn per sequence, ``num_return_sequences`` independent searches
        per prompt); it raises ``ValueError`` where 4.31 does, when a step leaves fewer than num_beams non-eos
        candidates.

        Under ``enable_decode_graphs()`` greedy decoding (with or without the penalty) replays one CUDA graph per token
        with the eager loop's tokens; nucleus sampling is graphed only after ``enable_decode_graphs(True,
        sampling=True)``, and then draws from the kernel's Philox stream instead of ``torch.multinomial`` (same
        distribution, different tokens for a given ``generator`` seed).  Beam search replays one graph per step when
        its sizes are within ``ops.beam_select_supported`` (else it runs the eager loop), with the eager loop's tokens
        except where two candidates' scores lie within a few fp32 ulps (the kernel's log-softmax sums in another
        order than ``torch.log_softmax``).  Beam sample is graphed under ``enable_decode_graphs(True, sampling=True)``
        within ``ops.beam_sample_supported``, with Philox draws like graphed nucleus sampling."""
        from . import ops
        eos_ids = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else [int(e) for e in eos_token_id])
        if num_beams > 1:
            beam_args = (text_ids, visual_output, num_image_per_seq, max_num_image, attention_mask, max_new_tokens,
                         eos_token_id, pad_token_id, min_length, repetition_penalty, num_beams, length_penalty,
                         num_return_sequences)
            V = self.text_decoder.head.weight.shape[0]
            graphs = self._decode_graphs is not None and text_ids.is_cuda and max_new_tokens > 0
            if use_nucleus_sampling:                                     # HF beam_sample
                if graphs and self._decode_graph_sampling and ops.beam_sample_supported(num_beams, len(eos_ids), V):
                    return self._graphed_beam_search(*beam_args, sampling=(temperature, top_p, generator))
                return self._beam_sample(*beam_args, temperature=temperature, top_p=top_p, generator=generator)
            if graphs and ops.beam_select_supported(num_beams, len(eos_ids), V):
                return self._graphed_beam_search(*beam_args)
            return self._beam_search(*beam_args)
        B, L = text_ids.shape
        if attention_mask is None:
            attention_mask = torch.ones((B, L), dtype=torch.long, device=text_ids.device)
        mm_embeds, cross, feats = self.prepare(text_ids, visual_output, num_image_per_seq, max_num_image)
        position_ids = (attention_mask.long().cumsum(-1) - 1).masked_fill(attention_mask == 0, 1)   # causal_lm_cascade.py:181-183
        graphed = (self._decode_graphs is not None and static_cache and text_ids.is_cuda and max_new_tokens > 0 and
                   (not use_nucleus_sampling or self._decode_graph_sampling))
        if graphed:
            mode = "sample" if use_nucleus_sampling else ("greedy" if repetition_penalty != 1.0 else None)
            return self._graphed_decode(mm_embeds, cross, feats, attention_mask, position_ids, max_new_tokens, eos_ids,
                                        pad_token_id, min_length, mode, repetition_penalty, temperature, top_p, generator)
        # the image-only half of the 10 cross-attention layers, once per call (PreparedVision)
        feats = self.mm_decoder.prepare_vision(feats)
        # pre-allocated per-layer caches appended in place (the reference's cat-per-token re-copies every layer's cache)
        past = self.mm_decoder.static_cache(B, L + max_new_tokens, dtype=mm_embeds.dtype, device=mm_embeds.device) if static_cache else None
        out = self.mm_decoder(inputs_embeds=mm_embeds, attention_mask=attention_mask, position_ids=position_ids,
                              past_key_values=past, vision_hidden_states=feats, cross_attention_mask=cross, use_cache=True,
                              return_dict=True)
        past = out.past_key_values
        logits = self.text_decoder.logits(out.last_hidden_state[:, -1:])
        new_ids = []
        finished = torch.zeros((B,), dtype=torch.bool, device=text_ids.device)
        mask = attention_mask
        last_cross = cross[:, -1:, :]
        pos = position_ids[:, -1:]
        for step_idx in range(max_new_tokens):
            scores = logits[:, -1].float()
            if repetition_penalty != 1.0 and new_ids:                    # HF RepetitionPenaltyLogitsProcessor
                prev = torch.stack(new_ids, dim=1)
                picked = scores.gather(1, prev)
                scores = scores.scatter(1, prev, torch.where(picked < 0, picked * repetition_penalty, picked / repetition_penalty))
            if step_idx < min_length and eos_ids:                        # HF MinLengthLogitsProcessor
                scores[:, eos_ids] = float("-inf")
            if use_nucleus_sampling:                                     # temperature, then top-p (HF warper order)
                scores = scores / temperature
                srt, idx = scores.sort(dim=-1, descending=False)
                drop = srt.softmax(-1).cumsum(-1) <= (1.0 - top_p)
                drop[:, -1] = False                                      # always keep the most likely token
                scores = scores.masked_fill(drop.scatter(1, idx, drop), float("-inf"))
                nxt = torch.multinomial(scores.softmax(-1), 1, generator=generator).squeeze(1)
            else:
                nxt = scores.argmax(-1)
            if eos_ids:
                nxt = torch.where(finished, torch.full_like(nxt, pad_token_id), nxt)
                for e in eos_ids:
                    finished = finished | (nxt == e)
            new_ids.append(nxt)
            mask = torch.cat([mask, torch.ones((B, 1), dtype=mask.dtype, device=mask.device)], dim=1)
            pos = pos + 1
            step = self.mm_decoder(inputs_embeds=self.mm_decoder.embed_tokens(nxt[:, None]), attention_mask=mask,
                                   position_ids=pos, past_key_values=past, vision_hidden_states=feats,
                                   cross_attention_mask=last_cross, use_cache=True, return_dict=True)
            past = step.past_key_values
            logits = self.text_decoder.logits(step.last_hidden_state)
        return torch.stack(new_ids, dim=1)

    @torch.no_grad()
    def _beam_search(self, text_ids, visual_output, num_image_per_seq, max_num_image, attention_mask, max_new_tokens,
                     eos_token_id, pad_token_id, min_length, repetition_penalty, num_beams, length_penalty, num_return,
                     sampling=None):
        """Beam search with the bookkeeping of HF ``GenerationMixin.beam_search`` + ``BeamSearchScorer`` (transformers
        4.31, the version the reference pins; ``early_stopping=False``, one beam group): log-softmax scores, logits
        processors on the log-probabilities, top ``max(2, 1 + n_eos) * num_beams`` candidates per sequence (the
        reference's own beam search, beam_search_monkey_patch.py:265-269: enough that ``num_beams`` of them are never
        eos), finished hypotheses ranked by ``sum_logprobs / len(generated) ** length_penalty``, a sequence is done once
        ``num_beams`` hypotheses are all at least as good as the best running beam could become.  The prompt is
        prefilled ONCE per sequence and its cache rows are replicated per beam; every step re-gathers the cache rows by
        beam index (``_reorder_cache``).

        ``sampling = (temperature, top_p, generator)`` runs 4.31's ``beam_sample`` instead (``_beam_sample_candidates``
        chooses the candidates): every beam starts at score 0, each sequence is expanded to ``num_return`` independent
        beam searches that return their best hypothesis, and a step with fewer than ``num_beams`` non-eos candidates
        raises ``ValueError`` as 4.31 does."""
        B0, L = text_ids.shape
        nb, dev = num_beams, text_ids.device
        expand = num_return if sampling is not None else 1
        B = B0 * expand                                                            # independent beam searches
        if attention_mask is None:
            attention_mask = torch.ones((B0, L), dtype=torch.long, device=dev)
        eos_ids = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else [int(e) for e in eos_token_id])
        mm_embeds, cross, feats = self.prepare(text_ids, visual_output, num_image_per_seq, max_num_image)
        position_ids = (attention_mask.long().cumsum(-1) - 1).masked_fill(attention_mask == 0, 1)   # causal_lm_cascade.py:181-183
        pre = self.mm_decoder.static_cache(B0, L, dtype=mm_embeds.dtype, device=dev)
        out = self.mm_decoder(inputs_embeds=mm_embeds, attention_mask=attention_mask, position_ids=position_ids,
                              past_key_values=pre, vision_hidden_states=feats, cross_attention_mask=cross, use_cache=True,
                              return_dict=True)
        rep = torch.arange(B0, device=dev).repeat_interleave(expand * nb)         # beam row -> prompt
        past = self.mm_decoder.static_cache(B * nb, L + max_new_tokens, dtype=mm_embeds.dtype, device=dev)
        for dst, src in zip(past, pre):
            dst.k[:, :L].copy_(src.k.index_select(0, rep)); dst.v[:, :L].copy_(src.v.index_select(0, rep)); dst.length = L
        del pre
        logits = self.text_decoder.logits(out.last_hidden_state[:, -1:]).index_select(0, rep)
        feats_b, last_cross = feats.index_select(0, rep), cross[:, -1:, :].index_select(0, rep)
        mask, pos = attention_mask.index_select(0, rep), position_ids[:, -1:].index_select(0, rep)

        beam_scores = torch.zeros((B, nb), dtype=torch.float32, device=dev)
        if sampling is None:
            beam_scores[:, 1:] = -1e9                                              # beam_sample starts every beam at 0
        beam_scores = beam_scores.view(-1)
        seqs = torch.zeros((B * nb, 0), dtype=torch.long, device=dev)              # generated ids per beam row
        hyps = [_BeamHypotheses(nb, length_penalty) for _ in range(B)]
        done = [False] * B
        n_cand = max(2, 1 + len(eos_ids)) * nb

        for step_idx in range(max_new_tokens):
            scores = torch.log_softmax(logits[:, -1].float(), dim=-1)
            if repetition_penalty != 1.0 and seqs.shape[1] > 0:
                picked = scores.gather(1, seqs)
                scores = scores.scatter(1, seqs, torch.where(picked < 0, picked * repetition_penalty, picked / repetition_penalty))
            if step_idx < min_length and eos_ids:
                scores[:, eos_ids] = float("-inf")
            V = scores.shape[-1]
            if sampling is None:
                top_s, top_i = (scores + beam_scores[:, None]).view(B, nb * V).topk(n_cand, dim=1, largest=True, sorted=True)
            else:
                top_s, top_i = _beam_sample_candidates(scores, beam_scores, B, nb, *sampling)
            top_s_h, top_i_h, seqs_h = top_s.tolist(), top_i.tolist(), seqs.tolist()   # one host round trip per step
            cur_len = seqs.shape[1] + 1
            nxt_scores = [[0.0] * nb for _ in range(B)]
            nxt_tokens = [[pad_token_id] * nb for _ in range(B)]
            nxt_rows = [[b * nb] * nb for b in range(B)]
            for b in range(B):
                if done[b]:
                    continue
                k = 0
                for rank, (sc, idx) in enumerate(zip(top_s_h[b], top_i_h[b])):
                    row, tok = b * nb + idx // V, idx % V
                    if tok in eos_ids:
                        if rank >= nb:
                            continue
                        hyps[b].add(seqs_h[row], sc)
                    else:
                        nxt_scores[b][k], nxt_tokens[b][k], nxt_rows[b][k] = sc, tok, row
                        k += 1
                    if k == nb:
                        break
                if k < nb and sampling is not None:
                    raise ValueError(f"At most {nb} tokens in {[i % V for i in top_i_h[b]]} can be equal to "
                                     f"`eos_token_id: {eos_ids}`. Make sure {[i % V for i in top_i_h[b]]} are corrected.")
                if len(hyps[b].beams) >= nb and hyps[b].worst >= top_s_h[b][0] / (cur_len ** length_penalty):
                    done[b] = True
            beam_scores = torch.tensor(nxt_scores, dtype=torch.float32, device=dev).view(-1)
            tok_t = torch.tensor(nxt_tokens, dtype=torch.long, device=dev).view(-1)
            row_t = torch.tensor(nxt_rows, dtype=torch.long, device=dev).view(-1)
            seqs = torch.cat([seqs.index_select(0, row_t), tok_t[:, None]], dim=1)
            if all(done) or step_idx == max_new_tokens - 1:
                break
            for c in past:                                                        # _reorder_cache
                n = c.length
                c.k[:, :n].copy_(c.k.index_select(0, row_t)[:, :n]); c.v[:, :n].copy_(c.v.index_select(0, row_t)[:, :n])
            mask = torch.cat([mask.index_select(0, row_t), torch.ones((B * nb, 1), dtype=mask.dtype, device=dev)], dim=1)
            pos = pos.index_select(0, row_t) + 1
            step = self.mm_decoder(inputs_embeds=self.mm_decoder.embed_tokens(tok_t[:, None]), attention_mask=mask, position_ids=pos,
                                   past_key_values=past, vision_hidden_states=feats_b, cross_attention_mask=last_cross,
                                   use_cache=True, return_dict=True)
            logits = self.text_decoder.logits(step.last_hidden_state)
        return _beam_finalize(hyps, done, seqs.tolist(), beam_scores.tolist(), num_return // expand, max_new_tokens,
                              pad_token_id, eos_ids).to(dev)

    def _beam_sample(self, *beam_args, temperature=1.0, top_p=1.0, generator=None):
        """HF 4.31 ``beam_sample`` in torch ops: ``_beam_search``'s loop with ``_beam_sample_candidates``."""
        return self._beam_search(*beam_args, sampling=(temperature, top_p, generator))

    @torch.no_grad()
    def _graphed_beam_search(self, text_ids, visual_output, num_image_per_seq, max_num_image, attention_mask,
                             max_new_tokens, eos_token_id, pad_token_id, min_length, repetition_penalty, num_beams,
                             length_penalty, num_return, sampling=None):
        """``_beam_search`` on one CUDA graph replay per step (``_GraphedDecoder`` in ``"beam"`` mode, or in
        ``"beam_sample"`` mode with ``sampling = (temperature, top_p, generator)``); same arguments, same finalize."""
        B, L = text_ids.shape
        nb = num_beams
        expand = num_return if sampling is not None else 1
        if attention_mask is None:
            attention_mask = torch.ones((B, L), dtype=torch.long, device=text_ids.device)
        eos_ids = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else [int(e) for e in eos_token_id])
        mm_embeds, cross, feats = self.prepare(text_ids, visual_output, num_image_per_seq, max_num_image)
        position_ids = (attention_mask.long().cumsum(-1) - 1).masked_fill(attention_mask == 0, 1)   # causal_lm_cascade.py:181-183
        mode = "beam" if sampling is None else "beam_sample"
        dec = self._decode_graph(mm_embeds, feats, max_new_tokens, eos_ids, pad_token_id, min_length, mode, nb, expand)
        st = dec.generate_beams(mm_embeds, cross, feats, attention_mask, position_ids, repetition_penalty, length_penalty,
                                *(sampling or ()))
        if st.get("error"):
            raise ValueError(f"At most {nb} tokens in the {2 * nb} sampled candidates of a sequence can be equal to "
                             f"`eos_token_id: {eos_ids}`: a step drew more than {nb} eos candidates")
        hyps = []
        for b in range(B * expand):                                        # the slots in insertion order
            meta, ids, sc = st["hyp_meta"][b].tolist(), st["hyp_ids"][b].tolist(), st["hyp_scores"][b].tolist()
            slots = sorted((m[1], j) for j, m in enumerate(meta) if m[0] >= 0)
            hyps.append(_BeamHypotheses(nb, length_penalty, [(sc[j], ids[j][:meta[j][0]]) for _, j in slots]))
        done = [bool(d) for d in st["done"].tolist()]
        return _beam_finalize(hyps, done, st["history"].tolist(), st["beam_scores"].tolist(), num_return // expand,
                              max_new_tokens, pad_token_id, eos_ids).to(text_ids.device)


_BEAM_SAMPLE_TOP_K = 50              # transformers 4.31 GenerationConfig.top_k, which the reference never overrides


def _beam_sample_candidates(scores, beam_scores, B, nb, temperature, top_p, generator):
    """Steps 3-5 of one 4.31 ``beam_sample`` step on the processed log-probabilities ``scores`` (B * nb, V): add the
    beam scores, warp (temperature, top-k 50, top-p; ``min_tokens_to_keep = 2``), draw ``2 * nb`` candidates per
    sequence with ``torch.multinomial`` (without replacement) and sort them by warped score.  Returns (scores, flat
    indices), each (B, 2 * nb)."""
    s = scores + beam_scores[:, None]
    if temperature != 1.0:                                                  # TemperatureLogitsWarper
        s = s / temperature
    V = s.shape[-1]
    k = min(max(_BEAM_SAMPLE_TOP_K, 2), V)                                  # TopKLogitsWarper
    s = s.masked_fill(s < s.topk(k, dim=-1).values[:, -1:], float("-inf"))
    if top_p < 1.0:                                                         # TopPLogitsWarper
        srt, idx = s.sort(dim=-1, descending=False)
        drop = srt.softmax(-1).cumsum(-1) <= (1.0 - top_p)
        drop[:, -2:] = False
        s = s.masked_fill(drop.scatter(1, idx, drop), float("-inf"))
    s = s.view(B, nb * V)
    pick = torch.multinomial(s.softmax(-1), 2 * nb, generator=generator)
    picked, order = s.gather(1, pick).sort(dim=1, descending=True, stable=True)   # ties: in draw order
    return picked, pick.gather(1, order)


class _BeamHypotheses:
    """The finished hypotheses of one sequence as HF's ``BeamHypotheses`` keeps them (``early_stopping=False``):
    ``(score, ids)`` in insertion order, at most ``num_beams``; a full set drops its first lowest-scored entry."""

    def __init__(self, num_beams, length_penalty, beams=()):
        self.num_beams, self.length_penalty = num_beams, length_penalty
        self.beams = list(beams)
        self.worst = min((h[0] for h in self.beams), default=1e9)

    def add(self, ids, sum_logprobs):
        score = sum_logprobs / (max(len(ids), 1) ** self.length_penalty)
        if len(self.beams) < self.num_beams or score > self.worst:
            self.beams.append((score, ids))
            if len(self.beams) > self.num_beams:
                self.beams.remove(min(self.beams, key=lambda h: h[0]))
            self.worst = min(h[0] for h in self.beams)


def _beam_finalize(hyps, done, seqs, beam_scores, num_return, max_new_tokens, pad_token_id, eos_ids):
    """End of beam search (eager and graphed): the running beams of unfinished sequences become hypotheses, the best
    ``num_return`` per sequence are returned as (B * num_return, width) ids on the CPU, padded with ``pad_token_id``
    after one ``eos_ids[0]``; width = min(longest + 1, max_new_tokens)."""
    nb = len(seqs) // len(hyps)
    for b, h in enumerate(hyps):
        if not done[b]:
            for j in range(nb):
                h.add(seqs[b * nb + j], beam_scores[b * nb + j])
    best = []
    for h in hyps:
        ranked = sorted(h.beams, key=lambda x: x[0])
        for _ in range(num_return):
            best.append(ranked.pop()[1])
    width = min(max(len(x) for x in best) + 1, max_new_tokens)
    out_ids = torch.full((len(best), width), pad_token_id, dtype=torch.long)
    for i, x in enumerate(best):
        out_ids[i, :len(x)] = torch.tensor(x, dtype=torch.long)
        if len(x) < width and eos_ids:
            out_ids[i, len(x)] = eos_ids[0]
    return out_ids


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
        (``pos_proj``, ``pos_ln``, ``post_ln``, the Q-Former, ``proj``); a trainable tokenizer encoder (CLIP ViT +
        ViT-Adapter) or an image loss raises up front, as neither has a backward here."""
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            if any(p.requires_grad for p in self.visual_tokenizer.encoder.parameters()):
                raise RuntimeError("MMInterleaved.forward under autograd: the visual tokenizer has no backward here "
                                   "through its CLIP ViT and ViT-Adapter; freeze them "
                                   "(model.visual_tokenizer.encoder.requires_grad_(False)) or run under torch.no_grad()")
            if self._has_image_loss():
                raise RuntimeError("MMInterleaved.forward under autograd: the image-decoder loss has no backward here; "
                                   "build the image decoder's VAE without an encoder (no image loss) or run under "
                                   "torch.no_grad()")
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

        The reference also trains the visual tokenizer's adapter and Q-Former head and the image decoder.  This leaves
        the tokenizer's flags as they are.  Its head (``pos_proj``, ``pos_ln``, ``post_ln``, the Q-Former, ``proj``) has
        a backward here, its encoder (CLIP ViT + ViT-Adapter) does not: ``forward`` under autograd raises while an
        encoder parameter requires grad or the image loss is on.  To train the text loss with the head trainable, freeze
        the encoder (``model.visual_tokenizer.encoder.requires_grad_(False)``); to train it without the tokenizer,
        freeze all of it (``model.visual_tokenizer.requires_grad_(False)``)."""
        for name, p in self.mm_decoder.named_parameters():
            p.requires_grad_("llama_cross_attn" in name)
        self.text_decoder.requires_grad_(False)
        self.text_decoder.head_new.requires_grad_(True)
        self.soi_token.requires_grad_(True)
        return self

    def _has_image_loss(self) -> bool:
        sd = getattr(self.image_decoder, "decoder", None)
        return getattr(getattr(sd, "vae", None), "encoder", None) is not None

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
