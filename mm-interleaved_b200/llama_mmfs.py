"""Llama decoder with injected MMFS cross-attention, H100-native.

Mirrors the module / parameter naming and the forward signatures of the reference's
``mm_interleaved/models/decoders/modeling_llama_mmfs.py`` (LlamaRMSNorm :53, LlamaMLP :175,
LlamaAttention :192, LlamaMMFSAttention :311, LlamaDecoderLayer :370, LlamaModel :562) so that a
reference checkpoint's state dict loads unchanged (``layers.N.self_attn.q_proj.weight`` ...), but
the forward is built for H100:

* q/k/v and gate/up projections run as ONE cuBLAS GEMM each on concatenated weights; o_proj and
  down_proj fold the residual add into the GEMM (``addmm``, beta = 1);
* RMSNorm, RoPE, SwiGLU and attention are hand-written sm_90a kernels (ops.py); q/k/v stay in the
  GEMM's (B, T, H, hd) layout -- no transposes, no materialised (B, H, T, T) score tensor, no
  additive 4-D mask (causality + key padding are applied inside the attention kernel);
* the MMFS cross-attention uses the fused sampler (mmfs.py); RMSNorm(vision) and
  value_proj(vision) are computed once per vision tensor and reused by every decode step
  (the reference recomputes both at each of the 10 cross layers at every generated token,
  SURVEY.md 3.2).

Plain library GEMMs (cuBLAS via torch) are used for the dense linears.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field
from types import SimpleNamespace
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from ._cache import SourceCache
from .mmfs import MMFS


@dataclass
class LlamaMMFSConfig:
    """The fields of HF ``LlamaConfig`` the reference reads, plus its three additions
    (cross_attention_frequency, spatial_shapes, image_embed_dim; mm_interleaved.py:300-304)."""
    vocab_size: int = 32002
    hidden_size: int = 5120
    intermediate_size: int = 13824
    num_hidden_layers: int = 40
    num_attention_heads: int = 40
    hidden_act: str = "silu"
    max_position_embeddings: int = 2048
    rms_norm_eps: float = 1e-6
    pad_token_id: int = 0
    cross_attention_frequency: int = 4
    spatial_shapes: List[int] = field(default_factory=lambda: [32, 16, 8])
    image_embed_dim: int = 1024
    use_cache: bool = True


class LlamaRMSNorm(nn.Module):
    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, hidden_states):
        return ops.rmsnorm(hidden_states.contiguous(), self.weight, self.variance_epsilon)


def rotary_tables(dim: int, max_pos: int, base: float = 10000.0, device=None):
    """cos / sin tables of FixedLlamaRotaryEmbedding (modeling_llama_mmfs.py:119-151), fp32 (max_pos, dim)."""
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2, device=device).float() / dim))
    t = torch.arange(max_pos, device=device, dtype=torch.float32)
    freqs = torch.outer(t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().contiguous(), emb.sin().contiguous()


_ROPE_TABLES = {}   # (device, head_dim) -> (n_positions, cos, sin); shared by every layer of every model on the device


def shared_rotary_tables(dim: int, need_pos: int, min_pos: int, device):
    """Tables covering at least ``need_pos`` positions.  One pair per (device, head_dim), grown geometrically: a decode
    loop that walks past ``max_position_embeddings`` must not rebuild 40 per-layer tables on every token (12 small
    kernels per layer per token in the round-2 decode profile).  Entries are prefixes of one another (row p depends on
    p only), so growing never changes a value a captured CUDA graph reads — but the graph holds the OLD storage, which
    the tuple below keeps alive only until it is replaced; graphed decoders therefore size the table once
    (need_pos = their static cache length) before capture."""
    key = (str(device), dim)
    hit = _ROPE_TABLES.get(key)
    if hit is None or hit[0] < need_pos:
        n = max(min_pos, need_pos if hit is None else max(need_pos, 2 * hit[0]))
        hit = (n,) + rotary_tables(dim, n, device=device)
        _ROPE_TABLES[key] = hit
    return hit[1], hit[2]


class _CatWeight:
    """Concatenation of several Linear weights along the output dim, rebuilt when a source changes."""

    def __init__(self, *linears):
        self.linears = linears
        self.key = None
        self.weight = None

    def get(self):
        key = tuple((l.weight.data_ptr(), l.weight._version, l.weight.dtype, l.weight.device) for l in self.linears)
        if key != self.key:
            with torch.no_grad():
                self.weight = torch.cat([l.weight for l in self.linears], 0).contiguous()
            self.key = key
        return self.weight


# Decode-step linears (at most 8 tokens in flight): ``ops.linear_skinny`` -- this repo's HBM-streaming kernel with the
# RMSNorm / SwiGLU in front folded in -- or cuBLAS + the stand-alone norm / activation kernel.  cuBLAS is the default
# (DESIGN.md section 4.7); MMFS_SKINNY_LINEARS=1 or ``llama_mmfs.SKINNY_DECODE_LINEARS = True`` switches.
SKINNY_DECODE_LINEARS = os.environ.get("MMFS_SKINNY_LINEARS", "0") == "1"


def _skinny(x, weight, prologue=0):
    return (SKINNY_DECODE_LINEARS and not torch.is_grad_enabled() and x.is_cuda and
            ops.linear_skinny_supported(x, weight, prologue))


def _addmm_residual(residual, x, weight, inplace):
    """residual + x @ weight^T as one GEMM with the residual as the beta = 1 accumulator.  ``torch.addmm`` out of
    place first copies the residual into the result (a D2D memcpy of the whole stream per call); in place skips it."""
    r2 = residual.view(-1, residual.shape[-1])
    x2 = x.reshape(-1, x.shape[-1])
    if inplace:
        r2.addmm_(x2, weight.t())
        return residual
    return torch.addmm(r2, x2, weight.t()).view_as(residual)


class LlamaMLP(nn.Module):
    def __init__(self, hidden_size: int, intermediate_size: int, hidden_act: str):
        super().__init__()
        if hidden_act != "silu":
            raise NotImplementedError("only the SiLU gate of Llama is implemented")
        self.gate_proj = nn.Linear(hidden_size, intermediate_size, bias=False)
        self.down_proj = nn.Linear(intermediate_size, hidden_size, bias=False)
        self.up_proj = nn.Linear(hidden_size, intermediate_size, bias=False)
        self._gate_up = _CatWeight(self.gate_proj, self.up_proj)

    def forward(self, x, residual=None, inplace=False, pre_norm=None):
        """``inplace``: accumulate into ``residual``'s storage (beta = 1 GEMM epilogue, no copy of the stream).
        ``pre_norm`` (extension): the LlamaRMSNorm in front of the block; ``x`` is then the un-normalised stream."""
        w_gu = self._gate_up.get()
        inter, hidden = self.down_proj.in_features, self.down_proj.out_features
        if pre_norm is not None and residual is not None and inplace and _skinny(x, w_gu, 1) and \
                ops.linear_skinny_shape_ok(x.shape[:-1].numel(), hidden, inter):           # down_proj's own limits
            gu = ops.linear_skinny(x, w_gu, norm_weight=pre_norm.weight, eps=pre_norm.variance_epsilon)
            ops.linear_skinny(gu, self.down_proj.weight, residual=residual, out=residual, swiglu=True)
            return residual
        if pre_norm is not None:
            x = pre_norm(x)
        gu = F.linear(x, w_gu)                                 # [gate | up] in one GEMM
        act = ops.swiglu(gu)
        if residual is None:
            return self.down_proj(act)
        return _addmm_residual(residual, act, self.down_proj.weight, inplace)


class StaticKV:
    """Pre-allocated key / value cache of one layer (extension): ``k``, ``v`` (B, T_max, H, hd) and the number of valid
    positions.  Passing it as ``past_key_value`` makes the layer append IN PLACE instead of the reference's
    ``torch.cat`` (modeling_llama_mmfs.py:236-239), which re-copies the whole cache of every layer for every token."""

    __slots__ = ("k", "v", "length", "slot")

    def __init__(self, batch, max_len, heads, head_dim, dtype, device):
        self.k = torch.empty((batch, max_len, heads, head_dim), dtype=dtype, device=device)
        self.v = torch.empty_like(self.k)
        self.length = 0
        # CUDA-graph decode (mm_interleaved.py::_GraphedGreedyDecoder): a (1,) int64 DEVICE tensor holding the slot the
        # next token is written to.  While set, a step appends at ``slot`` (index_copy_, no host integer involved),
        # attends over the WHOLE buffer under the caller's key mask, and ``length`` stays pinned at max_len - 1.
        self.slot = None


class PreparedVision:
    """Image-side state of the MMFS cross-attention layers for ONE batch of images: per layer, ``value`` =
    value_proj(RMSNorm(vision)) (modeling_llama_mmfs.py:353, mmfs.py:165-172) -- everything those layers derive from
    the images alone.  ``LlamaModel.prepare_vision`` fills it once; passing it as ``vision_hidden_states`` to prefill
    and to every decode step replaces the per-layer, per-token recomputation of the reference (and the implicit
    tensor-identity caches) by explicit scoping: the object lives exactly as long as its generate / forward call.
    With ``out=`` the values are written into existing storage (the static buffers a decode graph reads)."""

    __slots__ = ("raw_shape", "values")

    def __init__(self, raw_shape):
        self.raw_shape = tuple(raw_shape)        # (B, n_img, hw, C) of the packed feature tensor
        self.values = {}                          # layer index -> (B, n_img*hw, M, D)


class LlamaAttention(nn.Module):
    def __init__(self, config: LlamaMMFSConfig):
        super().__init__()
        self.config = config
        self.hidden_size = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.head_dim = self.hidden_size // self.num_heads
        self.max_position_embeddings = config.max_position_embeddings
        if self.head_dim * self.num_heads != self.hidden_size:
            raise ValueError("hidden_size must be divisible by num_heads")
        self.q_proj = nn.Linear(self.hidden_size, self.hidden_size, bias=False)
        self.k_proj = nn.Linear(self.hidden_size, self.hidden_size, bias=False)
        self.v_proj = nn.Linear(self.hidden_size, self.hidden_size, bias=False)
        self.o_proj = nn.Linear(self.hidden_size, self.hidden_size, bias=False)
        self._qkv = _CatWeight(self.q_proj, self.k_proj, self.v_proj)
        self._rope = None   # (device, max_pos, cos, sin)

    def rope_tables(self, device, need_pos):
        if self._rope is None or self._rope[0] != device or self._rope[1] < need_pos:
            cos, sin = shared_rotary_tables(self.head_dim, need_pos, self.max_position_embeddings, device)
            self._rope = (device, cos.shape[0], cos, sin)
        return self._rope[2], self._rope[3]

    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None,
                output_attentions=False, use_cache=False, residual=None, inplace=False, pre_norm=None):
        """``attention_mask``: (B, T_kv) key-padding mask, 1 = attend (what LlamaModel.forward receives,
        modeling_llama_mmfs.py:625) or None.  Causality is implicit (decoder).  Returns
        (attn_output [+ residual], None, present_key_value) like the reference (:217-280); the cache
        holds (key, value) in (B, T, H, hd) layout.  ``pre_norm`` (extension): the input LlamaRMSNorm;
        ``hidden_states`` is then the un-normalised stream (a decode step folds the norm into the q/k/v kernel)."""
        if output_attentions:
            raise NotImplementedError("attention probabilities are never materialised by the fused kernel")
        B, T, _ = hidden_states.shape
        H, hd = self.num_heads, self.head_dim
        w_qkv = self._qkv.get()
        skinny = _skinny(hidden_states, w_qkv, 1 if pre_norm is not None else 0)
        if skinny:
            qkv = ops.linear_skinny(hidden_states, w_qkv, norm_weight=None if pre_norm is None else pre_norm.weight,
                                    eps=0.0 if pre_norm is None else pre_norm.variance_epsilon).view(B, T, 3, H, hd)
        else:
            qkv = F.linear(hidden_states if pre_norm is None else pre_norm(hidden_states), w_qkv).view(B, T, 3, H, hd)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        static = isinstance(past_key_value, StaticKV)
        past = 0 if past_key_value is None else (past_key_value.length if static else past_key_value[0].shape[1])
        if position_ids is None:
            position_ids = torch.arange(past, past + T, device=hidden_states.device)
        cos, sin = self.rope_tables(hidden_states.device, past + T)
        if static and past_key_value.slot is not None:          # graph decode: device-side slot, whole buffer visible
            if T != 1:
                raise RuntimeError("StaticKV.slot (graph decode) takes one token per step")
            ops.rope_qk_append_(q, k, v, cos, sin, position_ids, past_key_value.k, past_key_value.v, past_key_value.slot)
            k, v = past_key_value.k, past_key_value.v
            past = k.shape[1] - 1
            present = past_key_value
        elif static:
            if past + T > past_key_value.k.shape[1]:
                raise RuntimeError(f"StaticKV of {past_key_value.k.shape[1]} positions cannot take {past} + {T}")
            ops.rope_qk_append_(q, k, v, cos, sin, position_ids, past_key_value.k, past_key_value.v, past)   # one kernel:
            past_key_value.length = past + T                                   # RoPE + both cache writes
            k, v = past_key_value.k[:, :past + T], past_key_value.v[:, :past + T]
            present = past_key_value
        else:
            ops.rope_qk_(q, k, cos, sin, position_ids)
            if past_key_value is not None:
                k = torch.cat([past_key_value[0], k], dim=1)
                v = torch.cat([past_key_value[1], v], dim=1)
            present = (k, v) if use_cache else None
        key_mask = None
        if attention_mask is not None:
            if attention_mask.dim() == 4:   # reference-style additive (B,1,T,T_kv): keys visible to the last query
                key_mask = attention_mask[:, 0, -1, :] > (torch.finfo(attention_mask.dtype).min / 2)
            else:
                key_mask = attention_mask
        ctx = ops.attention(q, k, v, key_mask=key_mask, causal=True, past=past)       # (B, T, H*hd)
        if skinny and residual is not None and inplace and _skinny(ctx, self.o_proj.weight):
            out = ops.linear_skinny(ctx, self.o_proj.weight, residual=residual, out=residual)
        else:
            out = self.o_proj(ctx) if residual is None else _addmm_residual(residual, ctx, self.o_proj.weight, inplace)
        return out, None, present


class LlamaMMFSAttention(nn.Module):
    def __init__(self, config: LlamaMMFSConfig, layer_idx):
        super().__init__()
        self.layer_idx = layer_idx
        self.config = config
        self.spatial_shapes = [(s, s) for s in config.spatial_shapes]
        self.hidden_size = config.hidden_size
        self.vision_hidden_size = config.image_embed_dim
        self.gate = nn.Parameter(torch.tensor([0.0]))
        self.attn = MMFS(layer_idx=layer_idx, d_model=self.hidden_size, d_query=self.hidden_size,
                         d_value=self.vision_hidden_size, d_out=self.hidden_size,
                         n_levels=len(config.spatial_shapes), n_heads=16, n_points=8,
                         ratio=self.vision_hidden_size / self.hidden_size, offset_init_magnitude=3.0,
                         spatial_shapes=config.spatial_shapes, max_num_image_per_seq=50)
        self.norm1 = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.norm2 = LlamaRMSNorm(self.vision_hidden_size, eps=config.rms_norm_eps)
        self._vision_cache = SourceCache()   # RMSNorm(vision features), identity-checked (see _cache.py)
        self._geom_cache = {}       # (device, n_img) -> (shapes, starts); (device, Lq) -> reference points

    def _geometry(self, device, n_img, hw, len_q):
        """deform_inputs (modeling_llama_mmfs.py:298-308) without its per-call host sync."""
        per_img = sum(h * w for h, w in self.spatial_shapes)
        if hw != per_img:
            raise RuntimeError(f"vision features have {hw} positions per image, expected {per_img}")
        key = ("s", device, n_img)
        if key not in self._geom_cache:
            ss = torch.tensor(self.spatial_shapes * n_img, dtype=torch.long)
            starts = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
            self._geom_cache[key] = (ss.to(device), starts.to(device))
        rkey = ("r", device, len_q)
        if rkey not in self._geom_cache:   # get_reference_points([(1,1)]): (0.5, 0.5) for every token (:306-307)
            self._geom_cache[rkey] = torch.full((1, len_q, 1, 2), 0.5, dtype=torch.float32, device=device)
        return self._geom_cache[key] + (self._geom_cache[rkey],)

    def _gated_output(self):
        """``output_proj`` pre-multiplied by tanh(gate) (:334 applies the gate to the block output), inference only."""
        w, b, g = self.attn.output_proj.weight, self.attn.output_proj.bias, self.gate
        key = (w.data_ptr(), w._version, b._version, g._version, w.dtype, w.device)
        if getattr(self, "_gated", None) is None or self._gated[0] != key:
            t = g.detach().float().tanh()
            self._gated = (key, (w.detach().float() * t).to(w.dtype), (b.detach().float() * t).to(b.dtype))
        return self._gated[1], self._gated[2]

    def project_vision(self, vision_hidden_states):
        """value_proj(RMSNorm(vision)) as (B, n_img*hw, M, D): the image-only part of this layer (:353, mmfs.py:165-172)."""
        return self.attn.project_value(self.norm2(vision_hidden_states))

    def forward(self, hidden_states, vision_hidden_states=None, cross_attention_mask=None, residual=None, inplace=False):
        h = self.norm1(hidden_states)
        value = None
        if isinstance(vision_hidden_states, PreparedVision):
            value = vision_hidden_states.values[self.layer_idx]
            _, n_img, hw, _ = vision_hidden_states.raw_shape
            v = None
        else:
            # RMSNorm(vision) depends only on the images: reuse it while the SAME tensor object is passed again (the
            # decode steps of one generate call); modeling_llama_mmfs.py:353 recomputes it per layer per token
            w2 = self.norm2.weight
            vextra = (w2.data_ptr(), w2._version)
            v = None if torch.is_grad_enabled() else self._vision_cache.get(vision_hidden_states, vextra)
            if v is None:
                v = self.norm2(vision_hidden_states)
                if not torch.is_grad_enabled():
                    self._vision_cache.put(vision_hidden_states, v, vextra)
            _, n_img, hw, _ = v.shape
        shapes, starts, ref = self._geometry(h.device, n_img, hw, h.shape[1])
        if not torch.is_grad_enabled():
            gw, gb = self._gated_output()
            out = self.attn(query=h, reference_points=ref, input_flatten=v, input_spatial_shapes=shapes,
                            input_level_start_index=starts, input_padding_mask=None, attention_mask=cross_attention_mask,
                            output_weight=gw, output_bias=gb, value=value)
            if residual is None:
                return out
            return residual.add_(out) if inplace else residual + out
        out = self.attn(query=h, reference_points=ref, input_flatten=v, input_spatial_shapes=shapes,
                        input_level_start_index=starts, input_padding_mask=None, attention_mask=cross_attention_mask,
                        value=value)
        gate = self.gate.tanh().to(out.dtype)
        if residual is None:
            return out * gate
        return torch.addcmul(residual, out, gate)


class LlamaDecoderLayer(nn.Module):
    def __init__(self, config: LlamaMMFSConfig, use_cross_attn: bool, layer_idx):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.self_attn = LlamaAttention(config=config)
        self.layer_idx = layer_idx
        self.llama_cross_attn = LlamaMMFSAttention(config=config, layer_idx=layer_idx) if use_cross_attn else None
        self.mlp = LlamaMLP(self.hidden_size, config.intermediate_size, config.hidden_act)
        self.input_layernorm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.post_attention_layernorm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)

    def forward(self, hidden_states, vision_hidden_states, cross_attention_mask, attention_mask=None,
                position_ids=None, past_key_value=None, output_attentions=False, use_cache=False, inplace=False):
        # norm -> self-attn -> (+) -> [MMFS cross-attn -> (+)] -> norm -> SwiGLU -> (+)   (:418-441)
        # ``inplace`` (extension, inference): the residual stream is updated in its own storage -- the caller
        # guarantees ``hidden_states`` is a private contiguous buffer (LlamaModel.forward clones the embeddings once).
        residual = hidden_states.contiguous()
        inplace = inplace and not torch.is_grad_enabled()
        hidden_states, _, present = self.self_attn(residual, attention_mask=attention_mask, position_ids=position_ids,
                                                   past_key_value=past_key_value, use_cache=use_cache, residual=residual,
                                                   inplace=inplace, pre_norm=self.input_layernorm)
        if self.llama_cross_attn is not None and vision_hidden_states is not None:
            hidden_states = self.llama_cross_attn(hidden_states, vision_hidden_states, cross_attention_mask,
                                                  residual=hidden_states, inplace=inplace)
        hidden_states = self.mlp(hidden_states, residual=hidden_states, inplace=inplace, pre_norm=self.post_attention_layernorm)
        outputs = (hidden_states,)
        if use_cache:
            outputs += (present,)
        return outputs


class LlamaModel(nn.Module):
    """Transformer decoder of ``config.num_hidden_layers`` layers with an MMFS cross-attention block in every
    ``cross_attention_frequency``-th layer (modeling_llama_mmfs.py:562-752)."""

    def __init__(self, config: LlamaMMFSConfig):
        super().__init__()
        self.config = config
        self.padding_idx = config.pad_token_id
        self.vocab_size = config.vocab_size
        self.cross_attention_frequency = config.cross_attention_frequency
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, self.padding_idx)
        use_cross = [i % self.cross_attention_frequency == 0 for i in range(config.num_hidden_layers)]
        self.layers = nn.ModuleList([LlamaDecoderLayer(config, use_cross[i], i) for i in range(config.num_hidden_layers)])
        self.norm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.gradient_checkpointing = False

    def static_cache(self, batch: int, max_len: int, dtype=None, device=None):
        """One ``StaticKV`` per layer, to be passed as ``past_key_values`` (prefill with length 0, then decode)."""
        p = self.embed_tokens.weight
        H = self.config.num_attention_heads
        return [StaticKV(batch, max_len, H, self.config.hidden_size // H, dtype or p.dtype, device or p.device)
                for _ in self.layers]

    @torch.no_grad()
    def prepare_vision(self, vision_hidden_states, out: Optional[PreparedVision] = None) -> PreparedVision:
        """Run the image-only part of every cross-attention layer once (see ``PreparedVision``)."""
        pv = PreparedVision(vision_hidden_states.shape) if out is None else out
        if tuple(vision_hidden_states.shape) != pv.raw_shape:
            raise RuntimeError(f"prepare_vision: features {tuple(vision_hidden_states.shape)} do not fit {pv.raw_shape}")
        for layer in self.layers:
            if layer.llama_cross_attn is None:
                continue
            val = layer.llama_cross_attn.project_vision(vision_hidden_states)
            if out is None:
                pv.values[layer.layer_idx] = val
            else:
                pv.values[layer.layer_idx].copy_(val)
        return pv

    def get_input_embeddings(self):
        return self.embed_tokens

    def set_input_embeddings(self, value):
        self.embed_tokens = value

    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                inputs_embeds=None, vision_hidden_states=None, cross_attention_mask=None, use_cache=None,
                output_attentions=None, output_hidden_states=None, return_dict=None):
        use_cache = self.config.use_cache if use_cache is None else use_cache
        return_dict = True if return_dict is None else return_dict
        if output_attentions:
            raise NotImplementedError("attention probabilities are never materialised")
        if input_ids is not None and inputs_embeds is not None:
            raise ValueError("You cannot specify both decoder_input_ids and decoder_inputs_embeds at the same time")
        if input_ids is None and inputs_embeds is None:
            raise ValueError("You have to specify either decoder_input_ids or decoder_inputs_embeds")
        if inputs_embeds is None:
            inputs_embeds = self.embed_tokens(input_ids)
        B, T, _ = inputs_embeds.shape
        if past_key_values is None:
            past = 0
        else:
            past = past_key_values[0].length if isinstance(past_key_values[0], StaticKV) else past_key_values[0][0].shape[1]
        if position_ids is None:
            position_ids = torch.arange(past, past + T, dtype=torch.long, device=inputs_embeds.device)
        else:
            position_ids = position_ids.view(-1, T).long()
        key_mask = None
        if attention_mask is not None:
            if tuple(attention_mask.shape) != (B, past + T):
                raise ValueError(f"attention_mask should be of size {(B, past + T)}, but is {tuple(attention_mask.shape)}")
            key_mask = attention_mask.to(torch.uint8)

        hidden_states = inputs_embeds
        inplace = not torch.is_grad_enabled() and not output_hidden_states
        if inplace:                      # one private copy of the stream; every layer then accumulates into it
            hidden_states = hidden_states.clone(memory_format=torch.contiguous_format)
        all_hidden = () if output_hidden_states else None
        next_cache = () if use_cache else None
        for idx, layer in enumerate(self.layers):
            if output_hidden_states:
                all_hidden += (hidden_states,)
            outs = layer(hidden_states, vision_hidden_states, cross_attention_mask, attention_mask=key_mask,
                         position_ids=position_ids,
                         past_key_value=past_key_values[idx] if past_key_values is not None else None,
                         use_cache=use_cache, inplace=inplace)
            hidden_states = outs[0]
            if use_cache:
                next_cache += (outs[1],)
        hidden_states = self.norm(hidden_states)
        if output_hidden_states:
            all_hidden += (hidden_states,)
        if not return_dict:
            return tuple(v for v in [hidden_states, next_cache, all_hidden] if v is not None)
        return SimpleNamespace(last_hidden_state=hidden_states, past_key_values=next_cache, hidden_states=all_hidden,
                               attentions=None)
