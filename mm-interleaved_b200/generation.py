"""Text generation of ``InterleavedForward.generate_texts``: the prompt setup every path shares, the eager token loop,
the eager beam loop (HF 4.31 ``beam_search`` and ``beam_sample``), and the CUDA-graphed decoders that
``enable_decode_graphs`` turns on (one graph replay per token or per beam step)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

from . import ops
from .llama_mmfs import PreparedVision, SharedPrefixKV, StaticKV, kv_storage

_BEAM_SAMPLE_TOP_K = 50              # transformers 4.31 GenerationConfig.top_k, which the reference never overrides


@dataclass
class Prompt:
    """What every decoding path needs from the call's inputs: the decoder inputs of the prompt, its (defaulted)
    attention mask, its position ids and the eos ids as a list.

    A prompt may continue a cached prefix (``interleaved.InterleavedSession``): ``cache`` (one ``StaticKV`` per layer)
    already holds its first ``prefix`` positions, so the prefill runs over the rest only, appending to ``cache``;
    ``vision`` is the ``PreparedVision`` of ``feats`` when the caller keeps one, and ``hidden`` (B, >= L, C), when given,
    receives the decoder's last hidden state of every prefilled position.  The decoding paths then start from the
    cached prompt instead of an empty cache, and leave ``cache`` at the prompt's length."""
    mm_embeds: torch.Tensor
    cross: torch.Tensor
    feats: torch.Tensor
    attention_mask: torch.Tensor
    position_ids: torch.Tensor
    eos_ids: List[int]
    cache: Optional[list] = None
    prefix: int = 0
    vision: Optional[PreparedVision] = None
    hidden: Optional[torch.Tensor] = None


def prepare_prompt(model, text_ids, visual_output, num_image_per_seq, max_num_image, attention_mask, eos_token_id):
    B, L = text_ids.shape
    if attention_mask is None:
        attention_mask = torch.ones((B, L), dtype=torch.long, device=text_ids.device)
    eos_ids = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else [int(e) for e in eos_token_id])
    mm_embeds, cross, feats = model.prepare(text_ids, visual_output, num_image_per_seq, max_num_image)
    position_ids = (attention_mask.long().cumsum(-1) - 1).masked_fill(attention_mask == 0, 1)   # causal_lm_cascade.py:181-183
    return Prompt(mm_embeds, cross, feats, attention_mask, position_ids, eos_ids)


def _prefill(model, p: Prompt, past, vision):
    """The decoder over the prompt's positions from ``p.prefix`` on into the cache ``past`` (which holds the ones
    before); returns (the cache, the last position's logits)."""
    s = p.prefix
    out = model.mm_decoder(inputs_embeds=p.mm_embeds[:, s:], attention_mask=p.attention_mask,
                           position_ids=p.position_ids[:, s:], past_key_values=past, vision_hidden_states=vision,
                           cross_attention_mask=p.cross[:, s:], use_cache=True, return_dict=True)
    if p.hidden is not None:
        p.hidden[:, s:p.mm_embeds.shape[1]].copy_(out.last_hidden_state)
    return out.past_key_values, model.text_decoder.logits(out.last_hidden_state[:, -1:])


def _prefill_beams(model, p: Prompt, rep, past, vision):
    """The prompt prefilled ONCE per sequence (into ``p.cache`` after its prefix, else into a fresh cache), its cache rows
    copied to the beam rows of ``past`` (``rep``: beam row -> prompt); returns the beam rows' last logits, attention
    mask, last position id and last cross-attention row."""
    B, L, _ = p.mm_embeds.shape
    pre = p.cache if p.cache is not None else \
        model.mm_decoder.static_cache(B, L, dtype=p.mm_embeds.dtype, device=p.mm_embeds.device, kv_fp8=model._kv_fp8)
    _, logits = _prefill(model, p, pre, vision)
    for dst, src in zip(past, pre):                                     # a copy of the prompt rows, no recompute
        dst.copy_rows_(src, rep, L)
        dst.length = L
    return (t.index_select(0, rep) for t in (logits, p.attention_mask, p.position_ids[:, -1:], p.cross[:, -1:, :]))


def generate_texts(model, text_ids, visual_output, num_image_per_seq, max_num_image, attention_mask, max_new_tokens,
                   eos_token_id, pad_token_id, static_cache, min_length, repetition_penalty, use_nucleus_sampling, top_p,
                   temperature, generator, num_beams, length_penalty, num_return_sequences):
    """``InterleavedForward.generate_texts``: one prompt setup, then ``decode``."""
    p = prepare_prompt(model, text_ids, visual_output, num_image_per_seq, max_num_image, attention_mask, eos_token_id)
    return decode(model, p, max_new_tokens, pad_token_id, static_cache, min_length, repetition_penalty,
                  use_nucleus_sampling, top_p, temperature, generator, num_beams, length_penalty, num_return_sequences)


def decode(model, p: Prompt, max_new_tokens, pad_token_id, static_cache, min_length, repetition_penalty,
           use_nucleus_sampling, top_p, temperature, generator, num_beams, length_penalty, num_return_sequences):
    """The graphed decoder where ``enable_decode_graphs`` is on and the kernels take the shape, else the eager loop."""
    if model._kv_fp8 and not static_cache:
        raise ValueError("static_cache=False keeps a 16-bit torch.cat cache: it cannot hold the FP8 KV cache that "
                         "enable_fp8_kv_cache() selects")
    V = model.text_decoder.head.weight.shape[0]
    graphs = (model._decode_graphs is not None and p.mm_embeds.is_cuda and max_new_tokens > 0 and
              (not use_nucleus_sampling or model._decode_graph_sampling))
    sample, warp = use_nucleus_sampling, (temperature, top_p, generator)
    if num_beams > 1:
        supported = ops.beam_sample_supported if sample else ops.beam_select_supported
        if graphs and supported(num_beams, len(p.eos_ids), V):
            dec = _graphed_decoder(model, p, max_new_tokens, pad_token_id, min_length, sample, num_beams,
                                   expand=num_return_sequences if sample else 1)
            return dec.generate(p, repetition_penalty, length_penalty, num_return_sequences, *warp)
        return beam_search(model, p, max_new_tokens, pad_token_id, min_length, num_beams, repetition_penalty,
                           length_penalty, num_return_sequences, sample, *warp)
    if graphs and static_cache and V <= ops.SELECT_MAX_V:
        dec = _graphed_decoder(model, p, max_new_tokens, pad_token_id, min_length, sample)
        return dec.generate(p, repetition_penalty, *warp)
    return token_loop(model, p, max_new_tokens, pad_token_id, static_cache, min_length, repetition_penalty, sample, *warp)


def token_loop(model, p: Prompt, max_new_tokens, pad_token_id, static_cache, min_length, repetition_penalty, sample,
               temperature, top_p, generator):
    """The eager single-sequence loop: prefill, then one decoder step per token with HF's processors in torch ops."""
    mm_embeds, attention_mask, eos_ids = p.mm_embeds, p.attention_mask, p.eos_ids
    B, L, _ = mm_embeds.shape
    # the image-only half of the 10 cross-attention layers, once per call (PreparedVision)
    feats = p.vision if p.vision is not None else model.mm_decoder.prepare_vision(p.feats)
    # pre-allocated per-layer caches appended in place (the reference's cat-per-token re-copies every layer's cache)
    if p.cache is not None:
        past = p.cache
    else:
        past = model.mm_decoder.static_cache(B, L + max_new_tokens, dtype=mm_embeds.dtype, device=mm_embeds.device,
                                             kv_fp8=model._kv_fp8) if static_cache else None
    past, logits = _prefill(model, p, past, feats)
    new_ids = []
    finished = torch.zeros((B,), dtype=torch.bool, device=mm_embeds.device)
    mask = attention_mask
    last_cross = p.cross[:, -1:, :]
    pos = p.position_ids[:, -1:]
    for step_idx in range(max_new_tokens):
        scores = logits[:, -1].float()
        if repetition_penalty != 1.0 and new_ids:                    # HF RepetitionPenaltyLogitsProcessor
            prev = torch.stack(new_ids, dim=1)
            picked = scores.gather(1, prev)
            scores = scores.scatter(1, prev, torch.where(picked < 0, picked * repetition_penalty, picked / repetition_penalty))
        if step_idx < min_length and eos_ids:                        # HF MinLengthLogitsProcessor
            scores[:, eos_ids] = float("-inf")
        if sample:                                                   # temperature, then top-p (HF warper order)
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
        step = model.mm_decoder(inputs_embeds=model.mm_decoder.embed_tokens(nxt[:, None]), attention_mask=mask,
                                position_ids=pos, past_key_values=past, vision_hidden_states=feats,
                                cross_attention_mask=last_cross, use_cache=True, return_dict=True)
        past = step.past_key_values
        logits = model.text_decoder.logits(step.last_hidden_state)
    if p.cache is not None:                                          # the generated positions are not kept
        for c in p.cache:
            c.length = L
    return torch.stack(new_ids, dim=1)


def beam_search(model, p: Prompt, max_new_tokens, pad_token_id, min_length, num_beams, repetition_penalty,
                length_penalty, num_return, sample, temperature, top_p, generator):
    """Beam search with the bookkeeping of HF ``GenerationMixin.beam_search`` + ``BeamSearchScorer`` (transformers
    4.31, the version the reference pins; ``early_stopping=False``, one beam group): log-softmax scores, logits
    processors on the log-probabilities, top ``max(2, 1 + n_eos) * num_beams`` candidates per sequence (the
    reference's own beam search, beam_search_monkey_patch.py:265-269: enough that ``num_beams`` of them are never
    eos), finished hypotheses ranked by ``sum_logprobs / len(generated) ** length_penalty``, a sequence is done once
    ``num_beams`` hypotheses are all at least as good as the best running beam could become.  The prompt is
    prefilled ONCE per sequence and its cache rows are replicated per beam; every step re-gathers the cache rows by
    beam index (``_reorder_cache``).

    ``sample`` runs 4.31's ``beam_sample`` instead (``_beam_sample_candidates`` chooses the candidates with
    ``temperature``, ``top_p`` and ``generator``): every beam starts at score 0, each sequence is expanded to
    ``num_return`` independent beam searches that return their best hypothesis, and a step with fewer than
    ``num_beams`` non-eos candidates raises ``ValueError`` as 4.31 does."""
    mm_embeds, eos_ids = p.mm_embeds, p.eos_ids
    B0, L, _ = mm_embeds.shape
    nb, dev = num_beams, mm_embeds.device
    expand = num_return if sample else 1
    B = B0 * expand                                                            # independent beam searches
    rep = torch.arange(B0, device=dev).repeat_interleave(expand * nb)         # beam row -> prompt
    past = model.mm_decoder.static_cache(B * nb, L + max_new_tokens, dtype=mm_embeds.dtype, device=dev,
                                         kv_fp8=model._kv_fp8)
    logits, mask, pos, last_cross = _prefill_beams(model, p, rep, past, p.vision if p.vision is not None else p.feats)
    feats_b = p.feats.index_select(0, rep)

    beam_scores = torch.zeros((B, nb), dtype=torch.float32, device=dev)
    if not sample:
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
        if not sample:
            top_s, top_i = (scores + beam_scores[:, None]).view(B, nb * V).topk(n_cand, dim=1, largest=True, sorted=True)
        else:
            top_s, top_i = _beam_sample_candidates(scores, beam_scores, B, nb, temperature, top_p, generator)
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
            if k < nb and sample:
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
            c.reorder_rows_(row_t, c.length)
        mask = torch.cat([mask.index_select(0, row_t), torch.ones((B * nb, 1), dtype=mask.dtype, device=dev)], dim=1)
        pos = pos.index_select(0, row_t) + 1
        step = model.mm_decoder(inputs_embeds=model.mm_decoder.embed_tokens(tok_t[:, None]), attention_mask=mask,
                                position_ids=pos, past_key_values=past, vision_hidden_states=feats_b,
                                cross_attention_mask=last_cross, use_cache=True, return_dict=True)
        logits = model.text_decoder.logits(step.last_hidden_state)
    return _beam_finalize(hyps, done, seqs.tolist(), beam_scores.tolist(), num_return // expand, max_new_tokens,
                          pad_token_id, eos_ids).to(dev)


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


def _graphed_decoder(model, p: Prompt, max_new_tokens, pad_id, min_length, sample, num_beams=1, expand=1):
    """The graphed decoder for this shape and these settings, built on first use (``model._decode_graphs`` keeps at
    most four); ``expand`` independent beam searches per prompt (beam sample's ``num_return_sequences``)."""
    B, L, _ = p.mm_embeds.shape
    B *= expand
    t_max = ((L + max_new_tokens + 255) // 256) * 256                  # cache-length bucket: one graph serves nearby prompts
    mode = ("beam_sample" if sample else "beam") if num_beams > 1 else ("sample" if sample else "greedy")
    key = (B, t_max, tuple(p.feats.shape), p.mm_embeds.dtype, p.mm_embeds.device, tuple(p.eos_ids), int(pad_id),
           int(min_length), int(max_new_tokens), bool(model._kv_fp8), int(num_beams), mode)
    dec = model._decode_graphs.get(key)
    if dec is None:
        if len(model._decode_graphs) >= 4:
            model._decode_graphs.pop(next(iter(model._decode_graphs)))
        args = (model, B, t_max, p.feats.shape, p.mm_embeds.dtype, p.mm_embeds.device, p.eos_ids, pad_id, min_length,
                max_new_tokens, sample)
        dec = model._decode_graphs[key] = BeamDecoder(*args, num_beams) if num_beams > 1 else TokenDecoder(*args)
    return dec


class _GraphedDecoder:
    """Static state + one CUDA graph of a decode step for ``InterleavedForward`` (see ``enable_decode_graphs``).

    Everything that changes from token to token lives in DEVICE tensors the graph updates itself -- the slot the new
    key/value row goes to, the key mask over the whole static cache, the position ids, the step counter, the finished
    flags, the chosen ids -- so generating N tokens is N ``graph.replay()`` calls with no host synchronisation.  The
    image-side tensors of the cross-attention layers are a ``PreparedVision`` over static storage, refilled eagerly once
    per call (a graph replay bypasses Python, so nothing inside the graph may depend on a tensor-identity cache).
    Per-call settings (penalties, temperature, top_p, seed) are device buffers too, so one graph serves any of their
    values.  A subclass sets ``past`` (the static caches of its R rows) and implements ``_choose``, the token choice
    of a step that writes ``next_ids``."""

    def __init__(self, model, B, R, t_max, feats_shape, dtype, device, eos_ids, pad_id, min_length, max_new, sample):
        self.owner, self.B, self.t_max, self.max_new, self.min_length = model, B, t_max, max_new, int(min_length)
        self.eos_ids, self.pad_id, self.sample = list(eos_ids), int(pad_id), bool(sample)
        self.pv = PreparedVision((R,) + tuple(feats_shape[1:]))
        probe = model.mm_decoder.prepare_vision(torch.zeros(feats_shape, dtype=dtype, device=device))
        for idx, val in probe.values.items():
            self.pv.values[idx] = val.new_empty((R,) + tuple(val.shape[1:]))
        V = model.text_decoder.head.weight.shape[0]
        self.logits = torch.zeros((R, V), dtype=torch.float32, device=device)
        self.key_mask = torch.zeros((R, t_max), dtype=torch.uint8, device=device)
        self.pos = torch.zeros((R, 1), dtype=torch.long, device=device)
        self.cur = torch.zeros((1,), dtype=torch.long, device=device)
        self.step = torch.zeros((1,), dtype=torch.long, device=device)
        self.finished = torch.zeros((B,), dtype=torch.bool, device=device)
        self.next_ids = torch.zeros((R, 1), dtype=torch.long, device=device)
        self.cross_last = torch.zeros((R, 1, feats_shape[1]), dtype=torch.float32, device=device)
        self.eos = torch.tensor(eos_ids, dtype=torch.long, device=device) if eos_ids else None
        self.seed = torch.zeros((1,), dtype=torch.long, device=device) if sample else None
        self.graph = None
        self.launches = 0
        self.replays = 0

    def _set_graph_mode(self, on: bool, length: int = 0):
        for c in self.past:
            c.slot = self.cur if on else None
            c.length = self.t_max - 1 if on else length

    def _start_call(self, L, generator, *params):
        """Per-call values the graph reads on the device: ``params`` in order and, when sampling, one seed per call."""
        if L + self.max_new > self.t_max:
            raise RuntimeError("prompt + new tokens exceed the captured cache length")
        for i, v in enumerate(params):
            self.params[i].fill_(float(v))
        if self.sample:                                                     # drawn on the device
            self.seed.random_(generator=generator)

    def _step(self):
        """One token: the token choice on the pending logits, then the decoder forward on the chosen token."""
        o = self.owner
        self._choose()
        self.key_mask.index_fill_(1, self.cur, 1)                          # the fed token's cache slot becomes visible
        self.pos.add_(1)
        hid = o.mm_decoder(inputs_embeds=o.mm_decoder.embed_tokens(self.next_ids), attention_mask=self.key_mask,
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
        self.cross_last.copy_(cross[:, -1:, :])
        self.logits.copy_(logits0)

    def _clear_unused(self, L):
        """Zero the cache positions from ``L`` on: masked slots must hold finite numbers."""
        for c in self.past:
            c.zero_from_(L)

    def _prefill_done(self, L, reset):
        """After the prefill: zero the unused cache slots, capture the step graph once, reset the per-call state."""
        self._clear_unused(L)
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
            self._captured_rope = [l.self_attn._rope for l in self.owner.mm_decoder.layers]
            self._clear_unused(L)                                           # the warm-up steps wrote the first new slot
        reset()

    def _replayed(self, L, n):
        """After ``n`` replays: count their launches and hand the caches back to eager use."""
        self.replays = n
        ops.launch_counter[0] += self.launches * n
        self._set_graph_mode(False, L)


class TokenDecoder(_GraphedDecoder):
    """One sequence per row: ``ops.decode_select`` chooses the token (greedy, with or without a repetition penalty,
    or temperature + top-p ``sample``), reading the penalty, temperature and top_p from ``params`` and, when
    sampling, one seed per call from ``seed``.  ``generate`` replays the graph ``max_new`` times."""

    def __init__(self, model, B, t_max, feats_shape, dtype, device, eos_ids, pad_id, min_length, max_new, sample):
        self.past = model.mm_decoder.static_cache(B, t_max, dtype=dtype, device=device, kv_fp8=model._kv_fp8)
        super().__init__(model, B, B, t_max, feats_shape, dtype, device, eos_ids, pad_id, min_length, max_new, sample)
        self.out_ids = torch.zeros((B, max_new), dtype=torch.long, device=device)
        self.params = torch.ones((3,), dtype=torch.float32, device=device)   # penalty, temperature, top_p

    def _choose(self):                                                     # processors, choice and bookkeeping: one kernel
        ops.decode_select(self.logits, self.out_ids, self.step, self.finished, self.next_ids, self.params, eos=self.eos,
                          pad_id=self.pad_id, min_length=self.min_length, sample=self.sample, seed=self.seed)

    def _reset(self, *args):
        super()._reset(*args)
        self.out_ids.fill_(self.pad_id)

    def generate(self, p: Prompt, repetition_penalty, temperature, top_p, generator):
        o = self.owner
        L = p.mm_embeds.shape[1]
        self._start_call(L, generator, repetition_penalty, temperature, top_p)
        o.mm_decoder.prepare_vision(p.feats, out=self.pv)                   # eager, into the static buffers the graph reads
        self._set_graph_mode(False, 0)
        if p.cache is None:
            _, logits = _prefill(o, p, self.past, self.pv)                  # prefill straight into the static cache
        else:                                                               # after a cached prefix: copy the prompt rows
            rows = torch.arange(p.mm_embeds.shape[0], device=p.mm_embeds.device)
            logits = next(_prefill_beams(o, p, rows, self.past, self.pv))
        logits0 = logits[:, -1].float()
        self._prefill_done(L, lambda: self._reset(L, p.attention_mask, p.position_ids, p.cross, logits0))
        for _ in range(self.max_new):
            self.graph.replay()
        self._replayed(L, self.max_new)
        return self.out_ids.clone()


class BeamDecoder(_GraphedDecoder):
    """Beam search over B * num_beams rows: the step is ``ops.beam_select`` (scores, hypotheses, done flags, history)
    -> ``ops.kv_beam_reorder`` (the generated positions of every layer's K and V, held in one tensor ``gen``) -> the
    decoder on the next tokens, with the repetition and length penalties in a device buffer; ``finished`` holds the
    per-sequence done flags.  With ``sample`` the step uses ``ops.beam_sample`` instead (temperature and top_p in the
    device buffer too, one seed per call, a sticky error flag) and every beam starts at score 0.

    The KV cache stores each prompt once: ``prefix`` (2·layers, P, T_p, H, hd), T_p = t_max - max_new, holds the P
    prompts' positions, which are the same for all G = R / P rows of a prompt (its beams, and with beam sample its
    independent searches); ``gen`` (2·layers, R, max_new, H, hd) holds every row's generated positions.  The decoder
    steps over ``SharedPrefixKV`` views of both (``ops.attention_decode_shared``)."""

    def __init__(self, model, B, t_max, feats_shape, dtype, device, eos_ids, pad_id, min_length, max_new, sample,
                 num_beams):
        nb = self.nb = int(num_beams)
        R = B * nb                                                          # decoder rows: one per beam
        P = feats_shape[0]                                                  # prompts: the features have one row each
        cfg, layers = model.mm_decoder.config, model.mm_decoder.layers
        n, H = 2 * len(layers), cfg.num_attention_heads
        hd = cfg.hidden_size // H
        fp8 = model._kv_fp8
        self.prefix, self.prefix_scale = kv_storage(n, P, t_max - max_new, H, hd, dtype, device, fp8)
        self.gen, self.gen_scale = kv_storage(n, R, max_new, H, hd, dtype, device, fp8)
        ps, gs = (self.prefix_scale, self.gen_scale) if fp8 else ([None] * n, [None] * n)
        self.prefix_kv = [StaticKV.over(self.prefix[2 * i], self.prefix[2 * i + 1], ps[2 * i], ps[2 * i + 1])
                          for i in range(len(layers))]
        self.prefix_len = torch.zeros((1,), dtype=torch.long, device=device)
        super().__init__(model, B, R, t_max, feats_shape, dtype, device, eos_ids, pad_id, min_length, max_new, sample)
        self.past = [SharedPrefixKV(self.prefix[2 * i], self.prefix[2 * i + 1], self.gen[2 * i], self.gen[2 * i + 1],
                                    self.prefix_len, self.step,
                                    (ps[2 * i], ps[2 * i + 1], gs[2 * i], gs[2 * i + 1]) if fp8 else None)
                     for i in range(len(layers))]
        # repetition_penalty, length_penalty (+ temperature, top_p when sampling)
        self.params = torch.ones((4 if sample else 2,), dtype=torch.float64, device=device)
        self.beam_scores = torch.zeros((R,), dtype=torch.float32, device=device)
        self.history = torch.zeros((R, max_new), dtype=torch.long, device=device)
        self.parent = torch.zeros((R,), dtype=torch.long, device=device)
        self.hyp_scores = torch.zeros((B, nb), dtype=torch.float64, device=device)
        self.hyp_ids = torch.zeros((B, nb, max_new), dtype=torch.long, device=device)
        self.hyp_meta = torch.zeros((B, nb, 2), dtype=torch.long, device=device)              # length (-1: free), serial
        n_scratch = ops.beam_sample_scratch(nb, R) if sample else R * ops.beam_candidates(nb, len(eos_ids))
        self.scratch = torch.zeros((n_scratch,), dtype=torch.long, device=device)
        self.all_done = torch.zeros((1,), dtype=torch.bool).pin_memory()                     # written by every replay
        if sample:
            self.error = torch.zeros((1,), dtype=torch.int32, device=device)

    def _choose(self):                                                     # scorer, then the cache follows the parents
        if self.sample:
            ops.beam_sample(self.logits, self.step, self.params, self.beam_scores, self.history, self.next_ids,
                            self.parent, self.finished, self.hyp_scores, self.hyp_ids, self.hyp_meta, self.error,
                            self.scratch, self.nb, eos=self.eos, pad_id=self.pad_id, min_length=self.min_length,
                            top_k=_BEAM_SAMPLE_TOP_K, seed=self.seed)
        else:
            ops.beam_select(self.logits, self.step, self.params, self.beam_scores, self.history, self.next_ids,
                            self.parent, self.finished, self.hyp_scores, self.hyp_ids, self.hyp_meta, self.scratch,
                            self.nb, eos=self.eos, pad_id=self.pad_id, min_length=self.min_length)
        ops.kv_beam_reorder(self.gen, self.parent, self.step, self.step, self.nb, self.max_new, done=self.finished)
        if self.gen_scale is not None:
            ops.kv_beam_reorder(self.gen_scale, self.parent, self.step, self.step, self.nb, self.max_new, done=self.finished)

    def _set_graph_mode(self, on: bool, length: int = 0):
        pass                                                               # SharedPrefixKV is graph-only: slot = step

    def _clear_unused(self, L):
        self.prefix[:, :, L:].zero_()
        self.gen.zero_()
        if self.gen_scale is not None:
            self.prefix_scale[:, :, L:].zero_()
            self.gen_scale.zero_()

    def _step(self):
        super()._step()
        self.all_done.copy_(self.finished.all().view(1), non_blocking=True)   # read by the host two replays later

    def _reset(self, *args):
        super()._reset(*args)
        if self.sample:
            self.beam_scores.zero_()                                       # beam_sample starts every beam at 0
            self.error.zero_()
        else:
            self.beam_scores.fill_(-1e9)
            self.beam_scores[::self.nb] = 0.0                              # only the first beam of a sequence is live
        self.history.fill_(self.pad_id)
        self.hyp_scores.zero_()
        self.hyp_meta.fill_(-1)

    def generate(self, p: Prompt, repetition_penalty, length_penalty, num_return, temperature, top_p, generator):
        """The prompt is prefilled once per sequence, straight into ``prefix`` (after an interleaved session's cached
        prefix: into the session's cache, whose B prompt rows are then copied), and the ``PreparedVision`` values, key
        mask, position ids and last cross-attention row are replicated to the beams (beam sample: to the ``self.B // B``
        independent searches of each prompt, then to their beams); then one replay per step.  At most two replays are
        in flight: before enqueuing replay t the host waits for replay t - 2 and reads the "all sequences done" flag it
        copied to pinned memory, so decoding stops at most two steps after the eager loop would (done sequences are
        inert).  The hypotheses are then rebuilt from the device slots and finalized as the eager loop does."""
        o = self.owner
        B, L, _ = p.mm_embeds.shape
        nb, expand = self.nb, self.B // B
        self._start_call(L, generator, repetition_penalty, length_penalty, *((temperature, top_p) if self.sample else ()))
        rep = torch.arange(B, device=p.mm_embeds.device).repeat_interleave(expand * nb)   # beam row -> prompt
        pv = o.mm_decoder.prepare_vision(p.feats)                           # the prefill's B rows, then one per beam
        for idx, val in pv.values.items():
            torch.index_select(val, 0, rep, out=self.pv.values[idx])
        for c in self.prefix_kv:
            c.length = 0
        if p.cache is None:
            _, logits = _prefill(o, p, self.prefix_kv, pv)
        else:
            logits = next(_prefill_beams(o, p, torch.arange(B, device=rep.device), self.prefix_kv, pv))
        del pv
        self.prefix_len.fill_(L)
        logits, mask_r, pos_r, cross_r = (t.index_select(0, rep) for t in (logits, p.attention_mask,
                                                                           p.position_ids[:, -1:], p.cross[:, -1:, :]))
        logits0 = logits[:, -1].float()
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
        self._replayed(L, n)
        if self.sample and bool(self.error.item()):
            raise ValueError(f"At most {nb} tokens in the {2 * nb} sampled candidates of a sequence can be equal to "
                             f"`eos_token_id: {self.eos_ids}`: a step drew more than {nb} eos candidates")
        meta_all, ids_all, sc_all = self.hyp_meta.tolist(), self.hyp_ids.tolist(), self.hyp_scores.tolist()
        hyps = []
        for meta, ids, sc in zip(meta_all, ids_all, sc_all):               # the slots in insertion order
            slots = sorted((m[1], j) for j, m in enumerate(meta) if m[0] >= 0)
            hyps.append(_BeamHypotheses(nb, length_penalty, [(sc[j], ids[j][:meta[j][0]]) for _, j in slots]))
        done = [bool(d) for d in self.finished.tolist()]
        return _beam_finalize(hyps, done, self.history[:, :n].tolist(), self.beam_scores.tolist(), num_return // expand,
                              self.max_new, self.pad_id, self.eos_ids).to(p.mm_embeds.device)
