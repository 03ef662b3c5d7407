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

    _PAD = 128   # a vocabulary of 32002+ rows is not a multiple of 8: cuBLAS drops to an unaligned legacy kernel (5x slower)

    def _fused(self):
        """head + head_new folded into one matrix / bias, rows zero-padded to a multiple of 128 (inference only)."""
        ps = (self.head.weight, self.head_new.weight, self.head.bias, self.head_new.bias)
        key = tuple((w.data_ptr(), w._version, w.dtype, w.device) for w in ps)
        if getattr(self, "_fused_cache", None) is None or self._fused_cache[0] != key:
            V, C = self.head.weight.shape
            Vp = (V + self._PAD - 1) // self._PAD * self._PAD
            with torch.no_grad():
                w = self.head.weight.new_zeros((Vp, C))
                w[:V] = self.head.weight
                w[self.orig_txt_vocab_size:V] += self.head_new.weight
                b = self.head.bias.new_zeros((Vp,))
                b[:V] = self.head.bias
                b[self.orig_txt_vocab_size:V] += self.head_new.bias
            self._fused_cache = (key, w, b)
        return self._fused_cache[1], self._fused_cache[2]

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
    schedule, sd.py:48-50) -- same attribute / state-dict names as the reference.  The VAE is a diffusers object this
    repository does not rebuild: ``vae_decode`` (a callable latents -> image in [-1, 1], e.g. ``AutoencoderKL.decode``)
    may be attached; without it ``generate_images`` returns the denoised latents (the pipeline's
    ``output_type="latent"`` result, sd.py:196-211)."""

    def __init__(self, unet=None, mmfs_module=None, image_size=512, base_seed=0, use_random_seed=False,
                 noise_scheduler=None, vae_decode=None, vae_scaling_factor=0.18215, **unet_kwargs):
        super().__init__()
        from . import unet_sd
        from .scheduler import DDPMScheduler, SD21_BASE_SCHEDULER
        self.unet = unet if unet is not None else unet_sd.UNet2DConditionModel(**unet_kwargs)
        self.mmfs_module = mmfs_module
        self.image_size, self.base_seed, self.use_random_seed = image_size, base_seed, use_random_seed
        self.noise_scheduler = noise_scheduler if noise_scheduler is not None else DDPMScheduler(**SD21_BASE_SCHEDULER)
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


class ImageDecoder(nn.Module):
    """``ImageDecoder`` (decoders/decoder_image.py:9-156): ``perceiver_resampler`` (Q-Former, 77 queries of width 1024
    over the per-image LLM context), ``neg_prompt_embeds`` and ``decoder`` = ``StableDiffusion`` (UNet + MMFSNet +
    scheduler).  State-dict names follow the reference (``decoder.unet.*``, ``decoder.mmfs_module.*``)."""

    def __init__(self, perceiver_config=None, seq_len=77, embed_dim=1024, unet=None, mmfs_module=None, image_size=512,
                 base_seed=0, sd_base_seed=None, sd_use_random_seed=False, mmfs_input_channel=1024, mmfs_feat_levels=4,
                 uncond_prob=0.1, decoder: Optional[nn.Module] = None, **_):
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
            decoder = StableDiffusion(unet=unet, mmfs_module=mmfs_module, image_size=image_size,
                                      base_seed=base_seed if sd_base_seed is None else sd_base_seed,
                                      use_random_seed=sd_use_random_seed)
        self.decoder = decoder

    # round-1 attribute names
    unet = property(lambda self: self.decoder.unet)
    mmfs_module = property(lambda self: self.decoder.mmfs_module)

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


class _GraphedGreedyDecoder:
    """Static state + one CUDA graph of a greedy decode step for ``InterleavedForward`` (see ``enable_decode_graphs``).

    Everything that changes from token to token lives in DEVICE tensors the graph updates itself -- the slot the new
    key/value row goes to, the key mask over the whole static cache, the position ids, the step counter, the finished
    flags, the output ids -- so generating N tokens is N ``graph.replay()`` calls with no host synchronisation.  The
    image-side tensors of the cross-attention layers are a ``PreparedVision`` over static storage, refilled eagerly once
    per call (a graph replay bypasses Python, so nothing inside the graph may depend on a tensor-identity cache)."""

    def __init__(self, owner, B, t_max, feats_shape, dtype, device, eos_ids, pad_id, min_length, max_new):
        from .llama_mmfs import PreparedVision
        self.owner, self.B, self.t_max, self.max_new, self.min_length = owner, B, t_max, max_new, int(min_length)
        model = owner.mm_decoder
        n_img = feats_shape[1]
        self.past = model.static_cache(B, t_max, dtype=dtype, device=device)
        self.pv = PreparedVision(feats_shape)
        probe = model.prepare_vision(torch.zeros(feats_shape, dtype=dtype, device=device))
        for idx, val in probe.values.items():
            self.pv.values[idx] = torch.empty_like(val)
        V = owner.text_decoder.head.weight.shape[0]
        self.logits = torch.zeros((B, V), dtype=torch.float32, device=device)
        self.key_mask = torch.zeros((B, t_max), dtype=torch.uint8, device=device)
        self.pos = torch.zeros((B, 1), dtype=torch.long, device=device)
        self.cur = torch.zeros((1,), dtype=torch.long, device=device)
        self.step = torch.zeros((1,), dtype=torch.long, device=device)
        self.finished = torch.zeros((B,), dtype=torch.bool, device=device)
        self.out_ids = torch.zeros((B, max_new), dtype=torch.long, device=device)
        self.cross_last = torch.zeros((B, 1, n_img), dtype=torch.float32, device=device)
        self.eos = torch.tensor(eos_ids, dtype=torch.long, device=device) if eos_ids else None
        self.pad = torch.tensor(int(pad_id), dtype=torch.long, device=device)
        self.neg_inf = torch.tensor(float("-inf"), dtype=torch.float32, device=device)
        self.zero = torch.zeros((), dtype=torch.float32, device=device)
        self.graph = None
        self.launches = 0

    def _set_graph_mode(self, on: bool, length: int = 0):
        for c in self.past:
            c.slot = self.cur if on else None
            c.length = self.t_max - 1 if on else length

    def _step(self):
        """One token: processors + arg-max on the pending logits, bookkeeping, decoder forward on the chosen token."""
        o = self.owner
        scores = self.logits
        if self.eos is not None and self.min_length > 0:                   # HF MinLengthLogitsProcessor
            bias = torch.where(self.step < self.min_length, self.neg_inf, self.zero)
            scores = scores.index_add(1, self.eos, bias.expand(self.B, self.eos.numel()).contiguous())
        nxt = scores.argmax(-1)
        if self.eos is not None:
            nxt = torch.where(self.finished, self.pad, nxt)
            self.finished.logical_or_((nxt[:, None] == self.eos[None, :]).any(dim=1))
        self.out_ids.index_copy_(1, self.step, nxt[:, None])
        self.key_mask.index_fill_(1, self.cur, 1)                          # the fed token's cache slot becomes visible
        self.pos.add_(1)
        hid = o.mm_decoder(inputs_embeds=o.mm_decoder.embed_tokens(nxt[:, None]), attention_mask=self.key_mask,
                           position_ids=self.pos, past_key_values=self.past, vision_hidden_states=self.pv,
                           cross_attention_mask=self.cross_last, use_cache=True, return_dict=True).last_hidden_state
        self.logits.copy_(o.text_decoder.logits(hid)[:, -1].float())
        self.step.add_(1)
        self.cur.add_(1)

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

    def generate(self, mm_embeds, cross, feats, attention_mask, position_ids):
        from . import ops
        o = self.owner
        B, L, _ = mm_embeds.shape
        if L + self.max_new > self.t_max:
            raise RuntimeError("prompt + new tokens exceed the captured cache length")
        o.mm_decoder.prepare_vision(feats, out=self.pv)                     # eager, into the static buffers the graph reads
        self._set_graph_mode(False, 0)
        out = o.mm_decoder(inputs_embeds=mm_embeds, attention_mask=attention_mask, position_ids=position_ids,
                           past_key_values=self.past, vision_hidden_states=self.pv, cross_attention_mask=cross,
                           use_cache=True, return_dict=True)               # prefill straight into the static cache
        logits0 = o.text_decoder.logits(out.last_hidden_state[:, -1:])[:, -1].float()
        for c in self.past:                                                 # masked slots must hold finite numbers
            c.k[:, L:].zero_()
            c.v[:, L:].zero_()
        self._set_graph_mode(True)
        if self.graph is None:
            self._reset(L, attention_mask, position_ids, cross, logits0)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):                                          # lazy handles, weight-derived caches, RoPE tables
                    self._reset(L, attention_mask, position_ids, cross, logits0)   # every warm-up step is step 0
                    self._step()
            torch.cuda.current_stream().wait_stream(side)
            self._reset(L, attention_mask, position_ids, cross, logits0)
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
        self._reset(L, attention_mask, position_ids, cross, logits0)
        for _ in range(self.max_new):
            self.graph.replay()
        ops.launch_counter[0] += self.launches * self.max_new
        self._set_graph_mode(False, L)
        return self.out_ids.clone()


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

    def enable_decode_graphs(self, enabled: bool = True) -> "InterleavedForward":
        """Greedy ``generate_texts`` then replays ONE captured CUDA graph per generated token (embedding -> 40 layers ->
        head -> logits processors -> arg-max -> state update, ~1000 kernels) instead of launching them from Python; the
        graph, its static KV cache and input buffers are kept per (batch, cache length, image count) and reused by
        later calls (SURVEY.md 8 f3; causal_lm_cascade.py:171-204 is the loop it replaces)."""
        self._decode_graphs = {} if enabled else None
        return self

    @torch.no_grad()
    def _graphed_greedy(self, mm_embeds, cross, feats, attention_mask, position_ids, max_new_tokens, eos_ids, pad_id, min_length):
        B, L, _ = mm_embeds.shape
        t_max = ((L + max_new_tokens + 255) // 256) * 256                  # cache-length bucket: one graph serves nearby prompts
        key = (B, t_max, tuple(feats.shape), mm_embeds.dtype, mm_embeds.device, tuple(eos_ids), int(pad_id), int(min_length),
               int(max_new_tokens))
        dec = self._decode_graphs.get(key)
        if dec is None:
            if len(self._decode_graphs) >= 4:
                self._decode_graphs.pop(next(iter(self._decode_graphs)))
            dec = self._decode_graphs[key] = _GraphedGreedyDecoder(self, B, t_max, feats.shape, mm_embeds.dtype, mm_embeds.device,
                                                                   eos_ids, pad_id, min_length, max_new_tokens)
        return dec.generate(mm_embeds, cross, feats, attention_mask, position_ids)

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
        (B * num_return_sequences, <= max_new_tokens) padded ids; otherwise (B, max_new_tokens) ids."""
        if num_beams > 1:
            if use_nucleus_sampling:
                raise NotImplementedError("beam-sample (num_beams > 1 with sampling) is not implemented")
            return self._beam_search(text_ids, visual_output, num_image_per_seq, max_num_image, attention_mask, max_new_tokens,
                                     eos_token_id, pad_token_id, min_length, repetition_penalty, num_beams, length_penalty,
                                     num_return_sequences)
        B, L = text_ids.shape
        if attention_mask is None:
            attention_mask = torch.ones((B, L), dtype=torch.long, device=text_ids.device)
        eos_ids = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else [int(e) for e in eos_token_id])
        mm_embeds, cross, feats = self.prepare(text_ids, visual_output, num_image_per_seq, max_num_image)
        position_ids = (attention_mask.long().cumsum(-1) - 1).masked_fill(attention_mask == 0, 1)   # causal_lm_cascade.py:181-183
        graphed = (self._decode_graphs is not None and static_cache and not use_nucleus_sampling and
                   repetition_penalty == 1.0 and text_ids.is_cuda and max_new_tokens > 0)
        if graphed:
            return self._graphed_greedy(mm_embeds, cross, feats, attention_mask, position_ids, max_new_tokens, eos_ids,
                                        pad_token_id, min_length)
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
                     eos_token_id, pad_token_id, min_length, repetition_penalty, num_beams, length_penalty, num_return):
        """Beam search with the bookkeeping of HF ``GenerationMixin.beam_search`` + ``BeamSearchScorer`` (transformers
        4.31, the version the reference pins; ``early_stopping=False``, one beam group): log-softmax scores, logits
        processors on the log-probabilities, top 2*num_beams candidates per sequence, finished hypotheses ranked by
        ``sum_logprobs / len(generated) ** length_penalty``, a sequence is done once ``num_beams`` hypotheses are all
        at least as good as the best running beam could become.  The prompt is prefilled ONCE per sequence and its
        cache rows are replicated per beam; every step re-gathers the cache rows by beam index (``_reorder_cache``)."""
        from .llama_mmfs import StaticKV
        B, L = text_ids.shape
        nb, dev = num_beams, text_ids.device
        if attention_mask is None:
            attention_mask = torch.ones((B, L), dtype=torch.long, device=dev)
        eos_ids = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else [int(e) for e in eos_token_id])
        mm_embeds, cross, feats = self.prepare(text_ids, visual_output, num_image_per_seq, max_num_image)
        position_ids = (attention_mask.long().cumsum(-1) - 1).masked_fill(attention_mask == 0, 1)   # causal_lm_cascade.py:181-183
        pre = self.mm_decoder.static_cache(B, L, dtype=mm_embeds.dtype, device=dev)
        out = self.mm_decoder(inputs_embeds=mm_embeds, attention_mask=attention_mask, position_ids=position_ids,
                              past_key_values=pre, vision_hidden_states=feats, cross_attention_mask=cross, use_cache=True,
                              return_dict=True)
        rep = torch.arange(B, device=dev).repeat_interleave(nb)                    # beam row -> sequence
        past = self.mm_decoder.static_cache(B * nb, L + max_new_tokens, dtype=mm_embeds.dtype, device=dev)
        for dst, src in zip(past, pre):
            dst.k[:, :L].copy_(src.k.index_select(0, rep)); dst.v[:, :L].copy_(src.v.index_select(0, rep)); dst.length = L
        del pre
        logits = self.text_decoder.logits(out.last_hidden_state[:, -1:]).index_select(0, rep)
        feats_b, last_cross = feats.index_select(0, rep), cross[:, -1:, :].index_select(0, rep)
        mask, pos = attention_mask.index_select(0, rep), position_ids[:, -1:].index_select(0, rep)

        beam_scores = torch.zeros((B, nb), dtype=torch.float32, device=dev)
        beam_scores[:, 1:] = -1e9
        beam_scores = beam_scores.view(-1)
        seqs = torch.zeros((B * nb, 0), dtype=torch.long, device=dev)              # generated ids per beam row
        hyps = [[] for _ in range(B)]                                              # per sequence: (score, ids list)
        worst = [1e9] * B
        done = [False] * B

        def add_hyp(b, ids, sum_logprobs):
            score = sum_logprobs / (max(len(ids), 1) ** length_penalty)
            if len(hyps[b]) < nb or score > worst[b]:
                hyps[b].append((score, ids))
                if len(hyps[b]) > nb:
                    hyps[b].remove(min(hyps[b], key=lambda h: h[0]))
                worst[b] = min(h[0] for h in hyps[b])

        for step_idx in range(max_new_tokens):
            scores = torch.log_softmax(logits[:, -1].float(), dim=-1)
            if repetition_penalty != 1.0 and seqs.shape[1] > 0:
                picked = scores.gather(1, seqs)
                scores = scores.scatter(1, seqs, torch.where(picked < 0, picked * repetition_penalty, picked / repetition_penalty))
            if step_idx < min_length and eos_ids:
                scores[:, eos_ids] = float("-inf")
            V = scores.shape[-1]
            cand = (scores + beam_scores[:, None]).view(B, nb * V)
            top_s, top_i = cand.topk(2 * nb, dim=1, largest=True, sorted=True)
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
                        add_hyp(b, seqs_h[row], sc)
                    else:
                        nxt_scores[b][k], nxt_tokens[b][k], nxt_rows[b][k] = sc, tok, row
                        k += 1
                    if k == nb:
                        break
                if len(hyps[b]) >= nb and worst[b] >= top_s_h[b][0] / (cur_len ** length_penalty):
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

        # finalize: running beams of unfinished sequences become hypotheses; best `num_return` per sequence
        seqs_h, bs_h = seqs.tolist(), beam_scores.tolist()
        for b in range(B):
            if not done[b]:
                for j in range(nb):
                    add_hyp(b, seqs_h[b * nb + j], bs_h[b * nb + j])
        best = []
        for b in range(B):
            ranked = sorted(hyps[b], key=lambda h: h[0])
            for _ in range(num_return):
                best.append(ranked.pop()[1])
        width = min(max(len(x) for x in best) + 1, max_new_tokens)
        out_ids = torch.full((len(best), width), pad_token_id, dtype=torch.long)
        for i, x in enumerate(best):
            out_ids[i, :len(x)] = torch.tensor(x, dtype=torch.long)
            if len(x) < width and eos_ids:
                out_ids[i, len(x)] = eos_ids[0]
        return out_ids.to(dev)


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
    text loss (and returns the logits) -- the image-decoder training loss needs the diffusers VAE and is not built;
    ``generate_images`` returns latents as ``image`` unless a ``vae_decode`` callable is attached to
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
        self.mm_decoder.gradient_checkpointing = use_llama_gradient_checkpointing      # inference: unused
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
        """mm_interleaved.py:408-518 up to the text loss.  Returns ``loss_txt`` / ``loss`` like the reference plus
        ``text_logits`` (B, T, V) (extension; ``return_loss=False`` stops there -- the "step" of SURVEY.md 8d).
        Inference-only kernels: call under ``torch.no_grad()``."""
        return_loss = kwargs.pop("return_loss", True)
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
        return out

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
