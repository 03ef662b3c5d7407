"""Interleaved image-text generation of one sample in one call (``MMInterleaved.generate_interleaved``): the turn loop
of the reference's ``inference.py::inference_all`` (:199-279) -- text turns through ``generate_texts``, image turns
through ``generate_images``, ``update_texts`` (:118-185) and ``update_image`` (:188-196) between them -- with the
state that never changes between turns kept on the device instead of recomputed.

Why keeping it is exact: the decoder is causal; a token cross-attends only to images whose ``<soi>`` precedes it
(``cross_attention_mask_from_ids``); an image's context is the hidden states of positions ``[0, soi]``
(``context_features_for_image_decoder``) and its MMFS features come from strictly earlier images
(``mmfs_features_for_image_decoder``).  So once a position is in the context, its keys, values and hidden state are
final, and so is every image's tokenizer output once the image is.  ``InterleavedSession`` keeps them:

* the visual tokenizer's outputs per image (each image is tokenized once; the grey placeholder of a pending image is
  not tokenized, as nothing reads it before the generated image replaces it -- except for a sample's first image,
  whose placeholder sizes the unread features as in the reference);
* one ``StaticKV`` per layer sized for the sample's final length, and the decoder's last hidden state per position;
* the ``PreparedVision`` of the current image set, rebuilt when an image is added.

A text turn prefills only the positions not yet cached, as one chunk after the cached prefix, and decodes from there
with the machinery of ``generation.py`` (eager or graphed, greedy, sampling, beam search, beam sample); the generated
ids are not kept in the cache (the next turn prefills them as part of its chunk, as the reference does).  An image
turn prefills the pending ids up to the target's ``<soi>``, builds the target's context and MMFS features with the
glue functions the forward uses, runs ``ImageDecoder.generate_images``, re-enters the first generated image with
``ops.image_reentry`` (bit-identical to the reference's PIL path, no host round trip) into the last image slot and
tokenizes that image alone; its 64 ``<image>`` positions are prefilled at the next text turn."""
from __future__ import annotations

import dataclasses
from typing import List, Optional

import torch

from . import generation, ops
from .mm_interleaved import context_features_for_image_decoder, mmfs_features_for_image_decoder

MODES = ("generate_texts", "generate_images")
TEXT_KWARGS = dict(max_length=30, min_length=8, num_beams=5, use_nucleus_sampling=False, top_p=0.9, temperature=1.0,
                   repetition_penalty=1.0, length_penalty=1.0)           # MMInterleaved.generate_texts' defaults
IMAGE_KWARGS = dict(guidance_scale=7.5, num_inference_steps=30, num_validation_images=1)   # ImageDecoder's


def update_texts(gen_ids: List[int], special_tokens: dict, num_img_token: int, force_gen_image_next: bool):
    """``update_texts`` (inference.py:118-185) on one text turn's ids: the first id dropped, a trailing ``<eos>`` removed
    (stop), ``<soi>`` appended when forced, ``num_img_token`` ``<image>`` ids after a final ``<soi>``.  Returns (the ids
    to append, whether an image turn follows, whether the text stopped)."""
    ids = list(gen_ids[1:])
    stopped = False
    if ids[-1] == special_tokens["eos_token_id"]:
        ids = ids[:-1]
        stopped = True
    if force_gen_image_next and ids[-1] != special_tokens["soi_token_id"]:
        ids.append(special_tokens["soi_token_id"])
    gen_image_next = ids[-1] == special_tokens["soi_token_id"]
    if gen_image_next:
        ids += [special_tokens["image_token_id"]] * num_img_token
    return ids, gen_image_next, stopped


def cache_budget(length: int, generate_mode: str, num_iter: int, max_length: int, num_img_token: int) -> int:
    """The most positions the sample can reach, over every outcome of its turns: a text turn decodes up to
    ``max_length`` positions past its prompt and appends at most ``max_length - 1`` ids (the first generated id is
    dropped), or, ending with a generated or forced ``<soi>``, at most ``max_length + num_img_token`` ids and hands the
    next turn to the image; an image turn appends nothing."""
    text, image = 0, 0                                  # most positions past the current ones, with k turns left
    for _ in range(max(num_iter, 0)):
        text, image = max(max_length, max_length - 1 + text, max_length + num_img_token + image), text
    return length + (image if generate_mode == "generate_images" else text)


def check_request(model, text_ids, attention_mask, image_tensors, num_image_per_seq, generate_mode,
                  force_replace_gen_text, kwargs):
    """The refusals, before any work: batch > 1, ``force_replace_gen_text`` (needs a text tokenizer), an unknown mode
    or keyword, an image decoder without a VAE decoder (the generated image could not re-enter the context)."""
    if text_ids.dim() != 2 or text_ids.shape[0] != 1 or image_tensors.dim() != 4 or num_image_per_seq.numel() != 1:
        raise ValueError("generate_interleaved generates one sample: text_ids (1, L), image_tensors (N, 3, R, R), "
                         f"one num_image_per_seq (got {tuple(text_ids.shape)}, {tuple(image_tensors.shape)}, "
                         f"{tuple(num_image_per_seq.shape)})")
    if attention_mask is not None and tuple(attention_mask.shape) != tuple(text_ids.shape):
        raise ValueError(f"attention_mask {tuple(attention_mask.shape)} does not match text_ids {tuple(text_ids.shape)}")
    if int(num_image_per_seq.reshape(-1)[0]) != image_tensors.shape[0]:
        raise ValueError("num_image_per_seq must count the sample's images")
    if force_replace_gen_text:
        raise NotImplementedError("force_replace_gen_text re-tokenizes text and needs a text tokenizer: not supported")
    if generate_mode not in MODES:
        raise ValueError(f"generate_mode must be one of {MODES}, got {generate_mode!r}")
    unknown = set(kwargs) - set(TEXT_KWARGS) - set(IMAGE_KWARGS)
    if unknown:
        raise TypeError(f"generate_interleaved: unexpected generation keywords {sorted(unknown)}")
    if int(kwargs.get("num_captions", 1)) != 1:
        raise ValueError("generate_interleaved keeps one text per turn")
    sd = getattr(getattr(model, "image_decoder", None), "decoder", None)
    if sd is None or getattr(sd, "vae_decode", None) is None:
        raise RuntimeError("generate_interleaved needs an image decoder with a VAE decoder (ImageDecoder(vae=True)): "
                           "a generated image re-enters the context as pixels")


class InterleavedSession:
    """The per-sample state of ``generate_interleaved`` (see the module docstring).  ``ids`` and ``mask`` are the
    sample's text ids (host list) and attention mask (device), ``images`` its (N, 3, R, R) fp32 image tensor, ``cached``
    the number of positions in ``cache`` / ``hidden``; ``tokenized`` counts the images the visual tokenizer has run on."""

    def __init__(self, model, text_ids, attention_mask, image_tensors, num_image_per_seq, capacity: int,
                 tokenize_last: bool = True):
        self.model = model
        self.st = model.special_token_dict
        dev = text_ids.device
        self.ids = [int(t) for t in text_ids[0].tolist()]
        self.mask = (torch.ones_like(text_ids) if attention_mask is None else attention_mask).to(dev).long()
        self.images = image_tensors.to(device=dev, dtype=torch.float32).contiguous().clone()
        self.n_img = int(num_image_per_seq.reshape(-1)[0])
        self.capacity = int(capacity)
        w = model.mm_decoder.embed_tokens.weight
        self.cache = model.mm_decoder.static_cache(1, self.capacity, dtype=w.dtype, device=dev)
        self.hidden = torch.zeros((1, self.capacity, w.shape[1]), dtype=w.dtype, device=dev)
        self.cached = 0
        self.vis_embed, self.ms = None, None
        self.tokenized = 0
        self.tokenizer_calls = 0
        self._pv, self._pv_key = None, None
        n = self.images.shape[0] - (0 if tokenize_last else 1)
        if n > 0:
            self._tokenize(self.images[:n])

    # ---- state --------------------------------------------------------------------------------------------------
    def _tokenize(self, images):
        out = self.model._tokenize(images)
        vis = out["vis_embed"].clone() if out.get("_static") else out["vis_embed"]
        ms = self.model._owned(out)
        if self.vis_embed is None:
            self.vis_embed, self.ms = vis, list(ms)
        else:
            self.vis_embed = torch.cat([self.vis_embed, vis])
            self.ms = [torch.cat([a, b]) for a, b in zip(self.ms, ms)]
        self.tokenized += images.shape[0]
        self.tokenizer_calls += 1

    def _ensure(self, need: int):
        if need > self.capacity:
            raise RuntimeError(f"interleaved session: {need} positions do not fit the cache of {self.capacity}")

    def _prompt(self, n: int, n_img: int, ms):
        """The ``Prompt`` of the first ``n`` ids over ``n_img`` image slots, continuing the cached prefix."""
        ids = torch.tensor([self.ids[:n]], dtype=torch.long, device=self.mask.device)
        vis = {"vis_embed": self.vis_embed, "multiscale_features": ms}
        nimg = torch.tensor([n_img], dtype=torch.long, device=ids.device)
        p = generation.prepare_prompt(self.model, ids, vis, nimg, n_img, self.mask[:, :n],
                                      [self.st.get("eos_token_id", 2), self.st["soi_token_id"]])
        key = (n_img, self.tokenizer_calls)                             # the image set the PreparedVision was built on
        if self._pv_key != key:
            self._pv, self._pv_key = None, None                         # release the old one first
            self._pv, self._pv_key = self.model.mm_decoder.prepare_vision(p.feats), key
        return ids, dataclasses.replace(p, cache=self.cache, prefix=self.cached, vision=self._pv, hidden=self.hidden)

    # ---- turns --------------------------------------------------------------------------------------------------
    def text_turn(self, kw, generator=None):
        """``generate_texts`` over the whole context: the uncached positions prefilled as one chunk, then decoding."""
        L = len(self.ids)
        self._ensure(L + kw["max_length"])
        if self.tokenized != self.n_img:
            raise RuntimeError("interleaved session: an image slot has no generated image yet")
        _, p = self._prompt(L, self.n_img, self.ms)
        out = generation.decode(self.model, p, kw["max_length"], self.st.get("pad_token_id", 0), True,
                                kw["min_length"], kw["repetition_penalty"], kw["use_nucleus_sampling"], kw["top_p"],
                                kw["temperature"], generator, kw["num_beams"], kw["length_penalty"], 1)
        self.cached = L
        return out

    def add_text(self, gen_ids: List[int], force_gen_image_next: bool):
        """``update_texts`` on the session: append the ids (and, for an image, a grey 0.5 placeholder slot)."""
        new, gen_image_next, stopped = update_texts(gen_ids, self.st, self.model.num_img_token, force_gen_image_next)
        self.ids += new
        self.mask = torch.cat([self.mask, self.mask.new_ones((1, len(new)))], dim=1)
        if gen_image_next:
            R = self.images.shape[-1]
            self.images = torch.cat([self.images, self.images.new_full((1, 3, R, R), 0.5)])
            self.n_img += 1
        return gen_image_next, stopped

    def image_turn(self, kw):
        """``generate_images`` of the last image slot, then ``update_image`` on the device."""
        n_tok = self.model.num_img_token
        soi = len(self.ids) - n_tok - 1
        if soi < 0 or self.ids[soi] != self.st["soi_token_id"] or self.tokenized != self.n_img - 1:
            raise RuntimeError("interleaved session: an image turn needs the text to end with <soi> and "
                               f"{n_tok} <image> ids of a pending image")
        n = soi + 1
        self._ensure(n)
        # The target slot's maps are never read: positions <= soi and the target itself see strictly earlier images
        # only.  Zeros stand in for them; with no earlier image, the placeholder's own maps do (as in the reference).
        placeholder = self.ms is None
        if placeholder:
            self._tokenize(self.images[-1:])
        ms = self.ms if placeholder else [torch.cat([f, f.new_zeros((1,) + tuple(f.shape[1:]))]) for f in self.ms]
        ids, p = self._prompt(n, self.n_img, ms)
        if self.cached < n:
            generation._prefill(self.model, p, self.cache, p.vision)
            self.cached = n
        m = self.model
        ctx, ctx_mask = context_features_for_image_decoder(self.hidden[:, :n], ids, self.st["soi_token_id"],
                                                           m.context_feat_proj, m.seq_len, self.n_img)
        feats, fmask = mmfs_features_for_image_decoder(ms, ids, self.st["soi_token_id"])
        out = m.image_decoder.generate_images(context_features=ctx[-1:], context_attention_mask=ctx_mask[-1:],
                                              mmfs_features=[f[-1:] for f in feats], mmfs_mask=fmask[-1:],
                                              num_inference_steps=kw["num_inference_steps"],
                                              guidance_scale=kw["guidance_scale"],
                                              num_validation_images=kw["num_validation_images"])
        images = out["image"]
        ops.image_reentry(images[:1].float(), self.images.shape[-1], out=self.images[-1:])
        if placeholder:
            self.vis_embed, self.ms, self.tokenized = None, None, 0
        self._tokenize(self.images[-1:])
        return images


def generate_interleaved(model, text_ids, image_tensors, num_image_per_seq, attention_mask=None,
                         generate_mode="generate_texts", num_iter=2, auto_end=False, force_gen_image_next=False,
                         force_replace_gen_text=False, generator: Optional[torch.Generator] = None,
                         max_cache_length: Optional[int] = None, return_session: bool = False, **kwargs):
    """``MMInterleaved.generate_interleaved``; returns ``turns`` (per turn, in order: ``{"mode": "generate_texts",
    "text_ids": ...}`` as ``generate_texts`` returns them, or ``{"mode": "generate_images", "image": ...}`` as
    ``generate_images`` does) and the final ``text_ids``, ``attention_mask``, ``image_tensors`` and
    ``num_image_per_seq`` as ``update_texts`` / ``update_image`` leave them; with ``return_session`` also the
    ``InterleavedSession`` (it holds the KV cache: drop it to free the memory)."""
    num_image_per_seq = num_image_per_seq.reshape(-1)
    check_request(model, text_ids, attention_mask, image_tensors, num_image_per_seq, generate_mode,
                  force_replace_gen_text, kwargs)
    kw = {**TEXT_KWARGS, **IMAGE_KWARGS, **kwargs}
    kw.pop("num_captions", None)
    budget = cache_budget(text_ids.shape[1], generate_mode, num_iter, kw["max_length"], model.num_img_token)
    if max_cache_length is not None and budget > max_cache_length:
        raise ValueError(f"generate_interleaved: the sample can reach {budget} positions, more than "
                         f"max_cache_length={max_cache_length}")
    dev = model.mm_decoder.embed_tokens.weight.device
    session = InterleavedSession(model, text_ids.to(dev), attention_mask, image_tensors, num_image_per_seq, budget,
                                 tokenize_last=generate_mode != "generate_images")
    turns = []
    mode = generate_mode
    stopped = False
    for _ in range(num_iter):
        if mode == "generate_texts":
            ids = session.text_turn(kw, generator)
            turns.append({"mode": mode, "text_ids": ids})
            gen_image_next, stopped = session.add_text(ids[0].tolist(), force_gen_image_next)
            if gen_image_next:
                mode = "generate_images"
        else:
            turns.append({"mode": mode, "image": session.image_turn(kw)})
            mode = "generate_texts"
        if auto_end and stopped:
            break
    ids = torch.tensor([session.ids], dtype=torch.long, device=dev)
    out = {"turns": turns, "text_ids": ids, "attention_mask": session.mask, "image_tensors": session.images,
           "num_image_per_seq": torch.tensor([session.n_img], dtype=torch.long, device=dev)}
    if return_session:
        out["session"] = session
    return out
