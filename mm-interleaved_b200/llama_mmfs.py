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
  SURVEY.md 3.2);
* the same modules carry the text loss's training path: RMSNorm, SwiGLU and attention go through the entry points of
  autograd_ops.py, which take the autograd Functions when autograd records the call and the inference kernels
  otherwise; ``LlamaAttention`` and ``LlamaMMFSAttention`` switch to their training forwards on ``msda.records``.

Plain library GEMMs (cuBLAS via torch) are used for the dense linears.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from types import SimpleNamespace
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

import torch.utils.checkpoint

from . import autograd_ops, ops
from ._cache import SourceCache, WeightCache
from .mmfs import MMFS
from .msda import records


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
        return autograd_ops.rmsnorm(hidden_states, self.weight, self.variance_epsilon)


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
    """Concatenation of several Linear weights along the output dim, rebuilt when a source changes; differentiable, and
    not cached, when autograd records a source weight (the cached copy is built without grad)."""

    def __init__(self, *linears):
        self.linears = linears
        self._cache = WeightCache()

    def get(self):
        ws = [l.weight for l in self.linears]
        if records(*ws):
            return torch.cat(ws, 0)
        return self._cache.get(ws, lambda: torch.cat(ws, 0).contiguous())


def _addmm_residual(residual, x, weight, inplace):
    """residual + x @ weight^T as one GEMM with the residual as the beta = 1 accumulator.  ``torch.addmm`` out of
    place first copies the residual into the result (a D2D memcpy of the whole stream per call); in place skips it."""
    r2 = residual.view(-1, residual.shape[-1])
    x2 = x.reshape(-1, x.shape[-1])
    if inplace:
        r2.addmm_(x2, weight.t())
        return residual
    return torch.addmm(r2, x2, weight.t()).view_as(residual)


# Where ops.linear_fp8 beat the bf16 cuBLAS GEMM on an H100 80GB HBM3 at 700 W (tools/fp8_decode_bench.py, DESIGN.md
# sections 4.9 and 6): at most 5 rows, and only the wide linears (N >= 2K: fused QKV, fused gate/up, the head).  At 20 rows and
# on o_proj / down_proj it was slower, so those calls keep the 16-bit weights.
FP8_DECODE_MAX_ROWS = 5


def decode_linear(x, weight, fp8, key, bias=None, residual=None, inplace=False):
    """``x @ weight^T [+ bias] [+ residual]``: the one place the decode-time linears (fused QKV, o_proj, fused gate/up,
    down_proj, the folded text head) choose their weights.  ``fp8`` is the module's ``WeightCache`` of FP8 copies while
    ``InterleavedForward.enable_fp8_decode`` is on, else None; ``key`` names the copy in it.  A decode-step call -- one
    position per row (x is (B, 1, K)), at most ``FP8_DECODE_MAX_ROWS`` rows, autograd not recording -- of a wide linear
    (N >= 2K, where the kernel wins) then runs ``ops.linear_fp8`` on the per-channel E4M3 copy of ``weight`` (``ops.quantize_fp8_per_channel``, built on first
    use and rebuilt when ``weight`` changes).  Every other call runs the 16-bit GEMM: ``F.linear``, or with
    ``residual`` the beta = 1 ``addmm`` (``inplace``: into ``residual``'s storage)."""
    if (fp8 is not None and x.dim() == 3 and x.shape[1] == 1 and x.shape[0] <= FP8_DECODE_MAX_ROWS
            and weight.shape[0] >= 2 * weight.shape[1] and not records(x, residual)):
        w8, scale = fp8.get(weight, lambda: ops.quantize_fp8_per_channel(weight), key)
        return ops.linear_fp8(x, w8, scale, bias, residual, out=residual if inplace else None)
    if residual is None:
        return F.linear(x, weight, bias)
    return _addmm_residual(residual, x, weight, inplace)


class LlamaMLP(nn.Module):
    def __init__(self, hidden_size: int, intermediate_size: int, hidden_act: str):
        super().__init__()
        if hidden_act != "silu":
            raise NotImplementedError("only the SiLU gate of Llama is implemented")
        self.gate_proj = nn.Linear(hidden_size, intermediate_size, bias=False)
        self.down_proj = nn.Linear(intermediate_size, hidden_size, bias=False)
        self.up_proj = nn.Linear(hidden_size, intermediate_size, bias=False)
        self._gate_up = _CatWeight(self.gate_proj, self.up_proj)
        self._fp8 = None                                       # FP8 decode copies (enable_fp8_decode)

    def forward(self, x, residual=None, inplace=False):
        """``inplace``: accumulate into ``residual``'s storage (beta = 1 GEMM epilogue, no copy of the stream)."""
        gu = decode_linear(x, self._gate_up.get(), self._fp8, "gate_up")       # [gate | up] in one GEMM
        act = autograd_ops.swiglu(gu)
        return decode_linear(act, self.down_proj.weight, self._fp8, "down", residual=residual, inplace=inplace)


class StaticKV:
    """Pre-allocated key / value cache of one layer (extension): ``k``, ``v`` (B, T_max, H, hd) and the number of valid
    positions.  Passing it as ``past_key_value`` makes the layer append IN PLACE instead of the reference's
    ``torch.cat`` (modeling_llama_mmfs.py:236-239), which re-copies the whole cache of every layer for every token.

    With ``kv_fp8`` (``InterleavedForward.enable_fp8_kv_cache``) ``k`` and ``v`` hold float8_e4m3fn bytes and
    ``k_scale`` / ``v_scale`` (B, T_max, ``ops.kv_scale_heads(H)``) fp32 one scale per (row, position, head)
    (``ops.quantize_kv_fp8``); for a 16-bit cache they are None.  The row operations below carry the scales along."""

    __slots__ = ("k", "v", "k_scale", "v_scale", "length", "slot")

    def __init__(self, batch, max_len, heads, head_dim, dtype, device, kv_fp8=False):
        kv, scales = kv_storage(2, batch, max_len, heads, head_dim, dtype, device, kv_fp8, torch.empty)
        self.k, self.v = kv[0], kv[1]
        self.k_scale, self.v_scale = (None, None) if scales is None else (scales[0], scales[1])
        self.length = 0
        # CUDA-graph decode (the graphed decoders of generation.py): a (1,) int64 DEVICE tensor holding the slot the
        # next token is written to.  While set, a step appends at ``slot`` (index_copy_, no host integer involved),
        # attends over the WHOLE buffer under the caller's key mask, and ``length`` stays pinned at max_len - 1.
        self.slot = None

    @classmethod
    def over(cls, k, v, k_scale=None, v_scale=None) -> "StaticKV":
        """An empty cache over existing (B, T_max, H, hd) storage, e.g. views of one tensor holding every layer's k and v
        (the graphed beam search reorders all of them in one launch)."""
        c = cls.__new__(cls)
        c.k, c.v, c.k_scale, c.v_scale, c.length, c.slot = k, v, k_scale, v_scale, 0, None
        return c

    @property
    def fp8(self) -> bool:
        return self.k_scale is not None

    def _tensors(self):
        if self.k_scale is None:
            return self.k, self.v
        return self.k.view(torch.uint8), self.v.view(torch.uint8), self.k_scale, self.v_scale   # bytes: moved as they are

    def copy_rows_(self, src: "StaticKV", rows: torch.Tensor, n: int) -> None:
        """Positions ``[:n]`` of row i become those of ``src``'s row ``rows[i]`` (the prompt's rows copied to its beams)."""
        if src.fp8 != self.fp8:
            raise RuntimeError("StaticKV.copy_rows_: an FP8 and a 16-bit cache do not mix")
        for dst, s in zip(self._tensors(), src._tensors()):
            dst[:, :n].copy_(s[:, :n].index_select(0, rows))

    def reorder_rows_(self, rows: torch.Tensor, n: int) -> None:
        """Positions ``[:n]`` of row i become those of row ``rows[i]`` (beam search's ``_reorder_cache``)."""
        for t in self._tensors():
            t[:, :n].copy_(t.index_select(0, rows)[:, :n])

    def zero_from_(self, n: int) -> None:
        """Zero positions ``n`` on: masked slots must hold finite numbers."""
        for t in self._tensors():
            t[:, n:].zero_()


def kv_storage(n, rows, max_len, heads, head_dim, dtype, device, kv_fp8=False, alloc=torch.zeros):
    """(data, scales) of ``n`` K or V caches in one tensor each (one launch of ``ops.kv_beam_reorder`` moves them all):
    data (n, rows, max_len, H, hd) of ``dtype``, or with ``kv_fp8`` float8_e4m3fn bytes and scales fp32
    (n, rows, max_len, ``ops.kv_scale_heads(H)``), else None."""
    data = alloc((n, rows, max_len, heads, head_dim), dtype=torch.float8_e4m3fn if kv_fp8 else dtype, device=device)
    if not kv_fp8:
        return data, None
    return data, torch.ones((n, rows, max_len, ops.kv_scale_heads(heads)), dtype=torch.float32, device=device)


class SharedPrefixKV:
    """Graph-decode cache of one layer whose rows come in groups of ``G`` that share a prompt (the graphed beam search,
    ``generation.BeamDecoder``): ``k``, ``v`` (P, T_p, H, hd) hold each prompt's positions once; ``k_gen``, ``v_gen``
    (P·G, max_new, H, hd) hold every row's generated positions.  Row r's position p lies in ``k[r // G, p]`` below
    ``prefix_len`` and in ``k_gen[r, p - prefix_len]`` from there on.  ``prefix_len`` and ``slot`` (where the next
    token's key / value go in ``k_gen``) are (1,) int64 DEVICE tensors, so one captured step serves every prompt length
    and step.  A step appends one token per row and attends over all ``length + 1`` = T_p + max_new positions under the
    caller's key mask (``ops.attention_decode_shared``); there is no eager use.

    An FP8 cache (``StaticKV``'s format) also carries the prefix's ``k_scale`` / ``v_scale`` and the generated
    positions' ``ks_gen`` / ``vs_gen``, and attends through ``ops.attention_decode_shared_fp8``."""

    __slots__ = ("k", "v", "k_gen", "v_gen", "G", "prefix_len", "slot", "k_scale", "v_scale", "ks_gen", "vs_gen")

    def __init__(self, k, v, k_gen, v_gen, prefix_len, slot, scales=None):
        self.k, self.v, self.k_gen, self.v_gen = k, v, k_gen, v_gen
        self.G = k_gen.shape[0] // k.shape[0]
        self.prefix_len, self.slot = prefix_len, slot
        self.k_scale, self.v_scale, self.ks_gen, self.vs_gen = scales if scales is not None else (None,) * 4

    @property
    def length(self):
        """Positions before the step's query, as ``StaticKV.length`` in graph decode (pinned at the last position)."""
        return self.k.shape[1] + self.k_gen.shape[1] - 1


class PrefixKV:
    """Read-only cache of one layer for scoring many short segments against one stored context
    (``MMInterleaved.enable_shared_context_scores``): ``k``, ``v`` (P, T_p, H, hd) are views of an existing cache's first
    T_p positions (e.g. ``StaticKV.k[:, :T_p]``), ``prefix_mask`` (P, T_p) marks the visible ones (or None), and the
    forward's T = G · ``seg_len`` positions per row are G segments.  A layer given it rotates its q and k at the explicit
    ``position_ids``, attends through ``ops.attention_prefix_shared`` (every visible prefix key, and causally the keys of
    the query's own segment) and appends nothing, so one prefill serves every segment; ``use_cache`` must be False."""

    __slots__ = ("k", "v", "prefix_mask", "seg_len")

    def __init__(self, k, v, prefix_mask, seg_len):
        self.k, self.v, self.prefix_mask, self.seg_len = k, v, prefix_mask, int(seg_len)


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


def _key_mask(attention_mask):
    """The (B, T_kv) key mask of a layer's ``attention_mask``: the mask itself, or of a reference-style additive
    (B, 1, T, T_kv) mask, the keys visible to the last query."""
    if attention_mask is None or attention_mask.dim() != 4:
        return attention_mask
    return attention_mask[:, 0, -1, :] > (torch.finfo(attention_mask.dtype).min / 2)


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
        self._fp8 = None    # FP8 decode copies (enable_fp8_decode)

    def rope_tables(self, device, need_pos):
        if self._rope is None or self._rope[0] != device or self._rope[1] < need_pos:
            cos, sin = shared_rotary_tables(self.head_dim, need_pos, self.max_position_embeddings, device)
            self._rope = (device, cos.shape[0], cos, sin)
        return self._rope[2], self._rope[3]

    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None,
                output_attentions=False, use_cache=False, residual=None, inplace=False):
        """``attention_mask``: (B, T_kv) key-padding mask, 1 = attend (what LlamaModel.forward receives,
        modeling_llama_mmfs.py:625) or None.  Causality is implicit (decoder).  Returns
        (attn_output [+ residual], None, present_key_value) like the reference (:217-280); the cache
        holds (key, value) in (B, T, H, hd) layout."""
        if output_attentions:
            raise NotImplementedError("attention probabilities are never materialised by the fused kernel")
        B, T, _ = hidden_states.shape
        H, hd = self.num_heads, self.head_dim
        if records(hidden_states, residual, self):
            return self._forward_training(hidden_states, attention_mask, position_ids, past_key_value, use_cache, residual)
        qkv = decode_linear(hidden_states, self._qkv.get(), self._fp8, "qkv").view(B, T, 3, H, hd)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        if isinstance(past_key_value, PrefixKV):
            return self._forward_prefix(q, k, v, position_ids, past_key_value, attention_mask, use_cache, residual,
                                        inplace)
        shared = isinstance(past_key_value, SharedPrefixKV)
        static = shared or isinstance(past_key_value, StaticKV)
        past = 0 if past_key_value is None else (past_key_value.length if static else past_key_value[0].shape[1])
        if position_ids is None:
            position_ids = torch.arange(past, past + T, device=hidden_states.device)
        cos, sin = self.rope_tables(hidden_states.device, past + T)
        key_mask = _key_mask(attention_mask)
        if static:
            # An FP8 cache (scales set): ops.rope_qk_append_fp8_ appends the rotated keys and the values as E4M3 and
            # rewrites the k / v views with x8 * scale, so every path below sees the keys and values x8 * scale.
            c, present = past_key_value, past_key_value
            fp8 = c.k_scale is not None
            if shared or c.slot is not None:                    # graph decode: device-side slot, whole buffer visible
                if T != 1:
                    raise RuntimeError("a graph-decode cache (SharedPrefixKV, StaticKV.slot) takes one token per step: "
                                       "prefill into a SharedPrefixKV's prefix through StaticKV.over")
                slot, n = c.slot, c.k.shape[1]
                if not shared:
                    past = n - 1
            else:
                if past + T > c.k.shape[1]:
                    raise RuntimeError(f"StaticKV of {c.k.shape[1]} positions cannot take {past} + {T}")
                slot, n = past, past + T
                c.length = n
            kc, vc, ksc, vsc = (c.k_gen, c.v_gen, c.ks_gen, c.vs_gen) if shared else (c.k, c.v, c.k_scale, c.v_scale)
            if fp8:
                ops.rope_qk_append_fp8_(q, k, v, cos, sin, position_ids, kc, vc, ksc, vsc, slot)
            else:
                ops.rope_qk_append_(q, k, v, cos, sin, position_ids, kc, vc, slot)    # one kernel: RoPE + both cache writes
            if shared and fp8:
                ctx = ops.attention_decode_shared_fp8(q, c.k, c.v, c.k_scale, c.v_scale, c.k_gen, c.v_gen, c.ks_gen,
                                                      c.vs_gen, c.prefix_len, key_mask=key_mask, past=past)
            elif shared:
                ctx = ops.attention_decode_shared(q, c.k, c.v, c.k_gen, c.v_gen, c.prefix_len, key_mask=key_mask,
                                                  past=past)
            elif fp8 and T == 1:
                ctx = ops.attention_decode_fp8(q, c.k[:, :n], c.v[:, :n], c.k_scale[:, :n], c.v_scale[:, :n],
                                               key_mask=key_mask, past=past)
            else:
                # 16-bit: the cache itself; an FP8 prefill from position 0: the rewritten k / v; after cached
                # positions: the cache's first n positions dequantised into a workspace
                if not fp8:
                    k, v = c.k[:, :n], c.v[:, :n]
                elif past > 0:
                    k = ops.kv_dequantize_fp8(c.k[:, :n], c.k_scale[:, :n], q.dtype)
                    v = ops.kv_dequantize_fp8(c.v[:, :n], c.v_scale[:, :n], q.dtype)
                ctx = ops.attention(q, k, v, key_mask=key_mask, causal=True, past=past)
        else:
            ops.rope_qk_(q, k, cos, sin, position_ids)
            if past_key_value is not None:
                k = torch.cat([past_key_value[0], k], dim=1)
                v = torch.cat([past_key_value[1], v], dim=1)
            present = (k, v) if use_cache else None
            ctx = ops.attention(q, k, v, key_mask=key_mask, causal=True, past=past)   # (B, T, H*hd)
        out = decode_linear(ctx, self.o_proj.weight, self._fp8, "o", residual=residual, inplace=inplace)
        return out, None, present

    def _forward_prefix(self, q, k, v, position_ids, c, attention_mask, use_cache, residual, inplace):
        """The layer over a ``PrefixKV``: RoPE on q and k at the explicit per-token ``position_ids`` (B, T), the
        prefix-shared attention with ``attention_mask`` (B, T) as the segments' own-key mask, o_proj; nothing is cached."""
        if use_cache:
            raise RuntimeError("PrefixKV is read-only: run the segments with use_cache=False")
        B, T = q.shape[:2]
        if position_ids is None or position_ids.numel() != B * T:
            raise RuntimeError("PrefixKV needs explicit position_ids of shape (B, T): the segments continue the prefix")
        cos, sin = self.rope_tables(q.device, c.k.shape[1] + c.seg_len)   # positions < T_p + seg_len (LlamaModel checks)
        ops.rope_qk_(q, k, cos, sin, position_ids)
        ctx = ops.attention_prefix_shared(q, c.k, c.v, k, v, c.seg_len, prefix_mask=c.prefix_mask, key_mask=attention_mask)
        return decode_linear(ctx, self.o_proj.weight, self._fp8, "o", residual=residual, inplace=inplace), None, None

    def _forward_training(self, hidden_states, attention_mask, position_ids, past_key_value, use_cache, residual):
        """The prefill under autograd: QKV GEMM -> RoPE -> causal attention (saving O and the row log-sum-exp) -> o_proj,
        each step with its backward (autograd_ops)."""
        if past_key_value is not None or use_cache:
            raise RuntimeError("LlamaAttention under autograd runs the prefill without a KV cache: pass use_cache=False "
                               "and no past_key_values, or run under torch.no_grad()")
        autograd_ops.check_training_dtype("LlamaAttention", hidden_states)
        if self.head_dim != 128:
            raise RuntimeError(f"LlamaAttention under autograd needs head dim 128 (the attention backward kernel's), "
                               f"got {self.head_dim}")
        B, T, _ = hidden_states.shape
        qkv = F.linear(hidden_states, self._qkv.get()).view(B, T, 3, self.num_heads, self.head_dim)
        if position_ids is None:
            position_ids = torch.arange(T, device=hidden_states.device)
        cos, sin = self.rope_tables(hidden_states.device, T)
        qkv = autograd_ops.rope_qkv(qkv, cos, sin, position_ids)
        ctx = autograd_ops.attention(qkv, _key_mask(attention_mask))
        out = self.o_proj(ctx) if residual is None else _addmm_residual(residual, ctx, self.o_proj.weight, False)
        return out, None, None


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
        self._gated = WeightCache()
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
        w, b, g = ps = self.attn.output_proj.weight, self.attn.output_proj.bias, self.gate

        def build():
            t = g.float().tanh()
            return (w.float() * t).to(w.dtype), (b.float() * t).to(b.dtype)
        return self._gated.get(ps, build)

    def project_vision(self, vision_hidden_states):
        """value_proj(RMSNorm(vision)) as (B, n_img*hw, M, D): the image-only part of this layer (:353, mmfs.py:165-172)."""
        return self.attn.project_value(self.norm2(vision_hidden_states))

    def forward(self, hidden_states, vision_hidden_states=None, cross_attention_mask=None, residual=None, inplace=False):
        if records(hidden_states, residual, vision_hidden_states, self):
            return self._forward_training(hidden_states, vision_hidden_states, cross_attention_mask, residual)
        h = self.norm1(hidden_states)
        value = None
        if isinstance(vision_hidden_states, PreparedVision):
            value = vision_hidden_states.values[self.layer_idx]
            _, n_img, hw, _ = vision_hidden_states.raw_shape
            v = None
        else:
            # RMSNorm(vision) depends only on the images: reuse it while the SAME tensor object is passed again (the
            # decode steps of one generate call); modeling_llama_mmfs.py:353 recomputes it per layer per token
            v = self._vision_cache.get_or_build((vision_hidden_states, self.norm2.weight),
                                                lambda: self.norm2(vision_hidden_states), cache=not torch.is_grad_enabled())
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

    def _forward_training(self, hidden_states, vision_hidden_states, cross_attention_mask, residual):
        """Under autograd: RMSNorms with their backward, then MMFS's differentiable path (front end in PyTorch, the
        gather through MSDeformAttnFunction) and the tanh gate."""
        if isinstance(vision_hidden_states, PreparedVision):
            raise RuntimeError("LlamaMMFSAttention under autograd takes the vision feature tensor, not PreparedVision "
                               "(an inference-only cache)")
        h = self.norm1(hidden_states)
        v = self.norm2(vision_hidden_states)
        _, n_img, hw, _ = v.shape
        shapes, starts, ref = self._geometry(h.device, n_img, hw, h.shape[1])
        out = self.attn.forward_differentiable(h, ref, v, shapes, starts, cross_attention_mask)
        out = out * self.gate.tanh().to(out.dtype)
        return out if residual is None else residual + out


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
        hidden_states, _, present = self.self_attn(self.input_layernorm(residual), attention_mask=attention_mask,
                                                   position_ids=position_ids, past_key_value=past_key_value,
                                                   use_cache=use_cache, residual=residual, inplace=inplace)
        if self.llama_cross_attn is not None and vision_hidden_states is not None:
            hidden_states = self.llama_cross_attn(hidden_states, vision_hidden_states, cross_attention_mask,
                                                  residual=hidden_states, inplace=inplace)
        hidden_states = self.mlp(self.post_attention_layernorm(hidden_states), residual=hidden_states, inplace=inplace)
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

    def static_cache(self, batch: int, max_len: int, dtype=None, device=None, kv_fp8: bool = False):
        """One ``StaticKV`` per layer, to be passed as ``past_key_values`` (prefill with length 0, then decode);
        ``kv_fp8``: E4M3 keys and values with per-head scales (see ``StaticKV``)."""
        p = self.embed_tokens.weight
        H = self.config.num_attention_heads
        return [StaticKV(batch, max_len, H, self.config.hidden_size // H, dtype or p.dtype, device or p.device, kv_fp8)
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
        training = records(inputs_embeds, vision_hidden_states, self)   # an embedding lookup below records through self
        if use_cache is None:   # under autograd the default is no cache, as HF's training path forces it
            use_cache = False if training else self.config.use_cache
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
        prefix = past_key_values is not None and isinstance(past_key_values[0], PrefixKV)
        if prefix:                     # segments over a read-only prefix: explicit positions, (B, T) own-key mask
            if use_cache:
                raise RuntimeError("PrefixKV is read-only: pass use_cache=False")
            if position_ids is None or position_ids.numel() != B * T:
                raise ValueError(f"past_key_values of PrefixKV need explicit position_ids of shape {(B, T)}")
            past = 0
        elif past_key_values is None:
            past = 0
        else:
            past = (past_key_values[0].length if isinstance(past_key_values[0], (StaticKV, SharedPrefixKV))
                    else past_key_values[0][0].shape[1])
        if position_ids is None:
            position_ids = torch.arange(past, past + T, dtype=torch.long, device=inputs_embeds.device)
        else:
            position_ids = position_ids.view(-1, T).long()
            if prefix:
                position_ids = position_ids.expand(B, T)
                limit = past_key_values[0].k.shape[1] + past_key_values[0].seg_len
                if int(position_ids.min()) < 0 or int(position_ids.max()) >= limit:
                    raise ValueError(f"PrefixKV segments sit at positions in [0, T_p + seg_len) = [0, {limit})")
        key_mask = None
        if attention_mask is not None:
            if tuple(attention_mask.shape) != (B, past + T):
                raise ValueError(f"attention_mask should be of size {(B, past + T)}, but is {tuple(attention_mask.shape)}")
            key_mask = attention_mask.to(torch.uint8)

        if training:
            if use_cache or past_key_values is not None:
                raise RuntimeError("LlamaModel under autograd runs the prefill without a KV cache: pass use_cache=False "
                                   "and no past_key_values, or run under torch.no_grad()")
            autograd_ops.check_training_dtype("LlamaModel", inputs_embeds)
        hidden_states = inputs_embeds
        inplace = not torch.is_grad_enabled() and not output_hidden_states
        if inplace:                      # one private copy of the stream; every layer then accumulates into it
            hidden_states = hidden_states.clone(memory_format=torch.contiguous_format)
        all_hidden = () if output_hidden_states else None
        next_cache = () if use_cache else None
        for idx, layer in enumerate(self.layers):
            if output_hidden_states:
                all_hidden += (hidden_states,)
            if training and self.gradient_checkpointing:   # activations recomputed in the backward, per layer (as HF)
                outs = torch.utils.checkpoint.checkpoint(layer, hidden_states, vision_hidden_states, cross_attention_mask,
                                                         attention_mask=key_mask, position_ids=position_ids,
                                                         use_reentrant=False)
            else:
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
