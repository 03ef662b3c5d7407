"""Tensor-level wrappers of the decoder-layer kernels (csrc/llama_ops_sm100.cu, csrc/attn_*.cu).

Host side is PyTorch (allocation, streams); every function enqueues exactly one hand-written kernel
through the C ABI and raises if the library rejects the arguments -- there is no PyTorch fallback.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import _lib
from .msda import _DTYPE_CODE, _require, inference_only

launch_counter = [0]   # kernels of ours launched through this module (bench.py's gpu_launches)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    """LlamaRMSNorm.forward (decoders/modeling_llama_mmfs.py:53-70) over the last dim."""
    inference_only("rmsnorm", x, weight)
    _require(x.is_cuda and x.is_contiguous() and weight.is_contiguous(), "rmsnorm: contiguous CUDA tensors required")
    _require(weight.dtype == x.dtype and weight.numel() == x.shape[-1], "rmsnorm: weight dtype / size mismatch")
    y = torch.empty_like(x)
    rows = x.numel() // x.shape[-1]
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_rmsnorm(x.data_ptr(), weight.data_ptr(), y.data_ptr(), rows, x.shape[-1], float(eps),
                                     _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "rmsnorm")
    launch_counter[0] += 1
    return y


def _check_affine(what: str, x: torch.Tensor, n: int, *params) -> None:
    """Optional per-channel weight / bias: the kernels read them as n contiguous elements of x's dtype."""
    for p in params:
        if p is not None:
            _require(p.dtype == x.dtype and p.numel() == n and p.is_contiguous() and p.device == x.device,
                     f"{what}: weight / bias must be contiguous {x.dtype} tensors of {n} elements on {x.device}")


def layernorm(x: torch.Tensor, weight, bias, eps: float) -> torch.Tensor:
    inference_only("layernorm", x, weight, bias)
    _require(x.is_cuda and x.is_contiguous(), "layernorm: contiguous CUDA tensor required")
    _check_affine("layernorm", x, x.shape[-1], weight, bias)
    y = torch.empty_like(x)
    rows = x.numel() // x.shape[-1]
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_layernorm(x.data_ptr(), weight.data_ptr() if weight is not None else None,
                                       bias.data_ptr() if bias is not None else None, y.data_ptr(), rows, x.shape[-1],
                                       float(eps), _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "layernorm")
    launch_counter[0] += 1
    return y


def rope_qk_(q: torch.Tensor, k: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, position_ids: torch.Tensor):
    """In-place rotary embedding of q and k, both (B, T, H, hd) views whose last two dims are dense
    (apply_rotary_pos_emb, decoders/modeling_llama_mmfs.py:165-172).  cos/sin: fp32 (max_pos, hd)."""
    B, T, H, hd = q.shape
    inference_only("rope_qk_", q, k)
    _require(q.is_cuda and k.shape == q.shape and q.stride(3) == 1 and q.stride(2) == hd and k.stride(3) == 1
             and k.stride(2) == hd and q.stride(0) == T * q.stride(1) and k.stride(0) == T * k.stride(1),
             "rope_qk_: q / k must be (B,T,H,hd) with dense heads and uniform token stride")
    _require(cos.dtype == torch.float32 and sin.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous()
             and cos.shape[-1] == hd, "rope_qk_: cos / sin must be contiguous fp32 (max_pos, hd)")
    pos = position_ids.to(torch.int64).contiguous()
    per_batch = 1 if pos.numel() == B * T else 0
    _require(per_batch or pos.numel() == T, "rope_qk_: position_ids must have B*T or T entries")
    with torch.cuda.device(q.device):
        rc = _lib.lib().mmfs_rope_qk(q.data_ptr(), k.data_ptr(), cos.data_ptr(), sin.data_ptr(), pos.data_ptr(),
                                     B * T, T, H, hd, q.stride(1), k.stride(1), per_batch, _DTYPE_CODE[q.dtype], _stream())
    _lib.check(rc, "rope_qk_")
    launch_counter[0] += 1


def rope_qk_append_(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor,
                    position_ids: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, slot) -> None:
    """``rope_qk_`` + the append to a static KV cache in one kernel: q rotated in place; rotated k and v of token t of
    batch entry b written to ``k_cache[b, slot + t]`` / ``v_cache[b, slot + t]``.  ``slot``: int (positions already
    cached) or a (1,) int64 CUDA tensor read by the kernel (graphed decode).  ``k`` itself is left unrotated."""
    B, T, H, hd = q.shape
    inference_only("rope_qk_append_", q, k, v)
    for t in (q, k, v):
        _require(t.is_cuda and tuple(t.shape) == (B, T, H, hd) and t.stride(3) == 1 and t.stride(2) == hd and
                 t.stride(0) == T * t.stride(1), "rope_qk_append_: q / k / v must be (B,T,H,hd) with dense heads and uniform token stride")
    for c in (k_cache, v_cache):
        _require(c.is_cuda and c.dim() == 4 and c.shape[0] == B and tuple(c.shape[2:]) == (H, hd) and c.stride(3) == 1 and
                 c.stride(2) == hd and c.dtype == q.dtype, "rope_qk_append_: caches must be (B, T_max, H, hd), dense heads")
    _require(k_cache.stride() == v_cache.stride(), "rope_qk_append_: k / v caches must share their strides")
    _require(cos.dtype == torch.float32 and sin.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous()
             and cos.shape[-1] == hd, "rope_qk_append_: cos / sin must be contiguous fp32 (max_pos, hd)")
    pos = position_ids.to(torch.int64).contiguous()
    per_batch = 1 if pos.numel() == B * T else 0
    _require(per_batch or pos.numel() == T, "rope_qk_append_: position_ids must have B*T or T entries")
    if isinstance(slot, torch.Tensor):
        _require(slot.is_cuda and slot.dtype == torch.int64 and slot.numel() == 1, "rope_qk_append_: slot tensor must be (1,) int64 on the device")
        slot_dev, slot_host = slot.data_ptr(), 0
    else:
        slot_dev, slot_host = None, int(slot)
        _require(0 <= slot_host and slot_host + T <= k_cache.shape[1], "rope_qk_append_: slot + T exceeds the cache")
    with torch.cuda.device(q.device):
        rc = _lib.lib().mmfs_rope_qk_append(q.data_ptr(), k.data_ptr(), v.data_ptr(), cos.data_ptr(), sin.data_ptr(), pos.data_ptr(),
                                            k_cache.data_ptr(), v_cache.data_ptr(), slot_dev, slot_host, B * T, T, H, hd,
                                            q.stride(1), k.stride(1), v.stride(1), k_cache.stride(0), k_cache.stride(1),
                                            per_batch, _DTYPE_CODE[q.dtype], _stream())
    _lib.check(rc, "rope_qk_append_")
    launch_counter[0] += 1


def decode_select(logits: torch.Tensor, out_ids: torch.Tensor, step: torch.Tensor, finished: torch.Tensor,
                  next_ids: torch.Tensor, params: torch.Tensor, eos: Optional[torch.Tensor] = None, pad_id: int = 0,
                  min_length: int = 0, sample: bool = False, seed: Optional[torch.Tensor] = None,
                  uniforms: Optional[torch.Tensor] = None) -> None:
    """One decode step's token choice in one kernel (csrc/decode_select_sm100.cu): HF's repetition penalty and
    min-length processors on the fp32 ``logits`` (B, V), then the arg-max or (``sample``) temperature + top-p sampling,
    then the finished / pad bookkeeping; the id is written to ``out_ids[:, step]`` and ``next_ids``.  ``step`` (1,)
    int64, ``params`` (3,) fp32 ``[repetition_penalty, temperature, top_p]`` and ``seed`` (1,) int64 are read on the
    device (a captured graph serves any of their values); ``finished`` (B,) bool / uint8 is updated in place;
    ``uniforms`` (B,) fp32 replaces the Philox draw when given."""
    inference_only("decode_select", logits)
    _require(logits.is_cuda and logits.dim() == 2 and logits.dtype == torch.float32 and logits.stride(1) == 1,
             "decode_select: logits must be a CUDA fp32 (B, V) tensor with unit column stride")
    B, V = logits.shape
    dev = logits.device
    _require(out_ids.device == dev and out_ids.dtype == torch.int64 and out_ids.dim() == 2 and out_ids.shape[0] == B
             and out_ids.is_contiguous(), "decode_select: out_ids must be contiguous int64 (B, max_new) on the logits' device")
    _require(step.device == dev and step.dtype == torch.int64 and step.numel() == 1, "decode_select: step must be a (1,) int64 device tensor")
    _require(finished.device == dev and finished.dtype in (torch.bool, torch.uint8) and finished.numel() == B
             and finished.is_contiguous(), "decode_select: finished must be contiguous bool / uint8 with B entries")
    _require(next_ids.device == dev and next_ids.dtype == torch.int64 and next_ids.numel() == B and next_ids.is_contiguous(),
             "decode_select: next_ids must be contiguous int64 with B entries")
    _require(params.device == dev and params.dtype == torch.float32 and params.numel() == 3 and params.is_contiguous(),
             "decode_select: params must be a contiguous (3,) fp32 device tensor [repetition_penalty, temperature, top_p]")
    if eos is not None:
        _require(eos.device == dev and eos.dtype == torch.int64 and eos.dim() == 1 and eos.is_contiguous(),
                 "decode_select: eos must be a contiguous 1-D int64 device tensor")
    if seed is not None:
        _require(seed.device == dev and seed.dtype == torch.int64 and seed.numel() == 1, "decode_select: seed must be a (1,) int64 device tensor")
    _require(not sample or seed is not None or uniforms is not None, "decode_select: sampling needs a seed or uniforms")
    if uniforms is not None:
        _require(uniforms.device == dev and uniforms.dtype == torch.float32 and uniforms.numel() == B and uniforms.is_contiguous(),
                 "decode_select: uniforms must be contiguous fp32 with B entries")
    seed_ptr = seed.data_ptr() if seed is not None else None
    with torch.cuda.device(dev):
        rc = _lib.lib().mmfs_decode_select(logits.data_ptr(), logits.stride(0), out_ids.data_ptr(), step.data_ptr(),
                                           finished.data_ptr(), next_ids.data_ptr(), eos.data_ptr() if eos is not None else None,
                                           eos.numel() if eos is not None else 0, int(pad_id), int(min_length),
                                           params.data_ptr(), seed_ptr, uniforms.data_ptr() if uniforms is not None else None,
                                           B, V, out_ids.shape[1], _lib.SELECT_SAMPLE if sample else _lib.SELECT_GREEDY,
                                           _stream())
    _lib.check(rc, "decode_select")
    launch_counter[0] += 1


SELECT_MAX_V = 1 << 17   # the vocabulary limit of decode_select, beam_select and beam_sample (kMaxV: two V-bit maps)


def beam_candidates(num_beams: int, n_eos: int) -> int:
    """Candidates per sequence of one beam step, the reference's ``max(2, 1 + n_eos) * num_beams``."""
    return max(2, 1 + n_eos) * num_beams


def beam_select_supported(num_beams: int, n_eos: int, V: int) -> bool:
    """Whether ``beam_select`` takes this shape (its limits: num_beams <= 8, n_eos <= 4, the candidates fit in V)."""
    return (1 <= num_beams <= _lib.BEAM_MAX_BEAMS and 0 <= n_eos <= _lib.BEAM_MAX_EOS
            and beam_candidates(num_beams, n_eos) <= V <= SELECT_MAX_V)


def _check_beam_step(what, logits, step, params, n_params, beam_scores, history, next_ids, parent, done, hyp_scores,
                     hyp_ids, hyp_meta, num_beams, eos):
    """The buffer checks ``beam_select`` and ``beam_sample`` share; returns (B, V, max_new, n_eos)."""
    inference_only(what, logits)
    _require(logits.is_cuda and logits.dim() == 2 and logits.dtype == torch.float32 and logits.stride(1) == 1,
             f"{what}: logits must be a CUDA fp32 (R, V) tensor with unit column stride")
    R, V = logits.shape
    dev = logits.device
    _require(num_beams > 0 and R % num_beams == 0, f"{what}: the rows must be whole groups of num_beams")
    B = R // num_beams

    def dense(t, name, dtype, shape):
        _require(t.device == dev and t.dtype == dtype and tuple(t.shape) == shape and t.is_contiguous(),
                 f"{what}: {name} must be a contiguous {dtype} {shape} tensor on the logits' device")

    _require(history.dim() == 2, f"{what}: history must be (R, max_new)")
    max_new = history.shape[1]
    dense(step, "step", torch.int64, (1,))
    dense(params, "params", torch.float64, (n_params,))
    dense(beam_scores, "beam_scores", torch.float32, (R,))
    dense(history, "history", torch.int64, (R, max_new))
    dense(next_ids, "next_ids", torch.int64, tuple(next_ids.shape))
    _require(next_ids.numel() == R, f"{what}: next_ids must have R entries")
    dense(parent, "parent", torch.int64, (R,))
    _require(done.device == dev and done.dtype in (torch.bool, torch.uint8) and done.numel() == B and done.is_contiguous(),
             f"{what}: done must be contiguous bool / uint8 with B entries")
    dense(hyp_scores, "hyp_scores", torch.float64, (B, num_beams))
    dense(hyp_ids, "hyp_ids", torch.int64, (B, num_beams, max_new))
    dense(hyp_meta, "hyp_meta", torch.int64, (B, num_beams, 2))
    n_eos = 0
    if eos is not None:
        _require(eos.device == dev and eos.dtype == torch.int64 and eos.dim() == 1 and eos.is_contiguous(),
                 f"{what}: eos must be a contiguous 1-D int64 device tensor")
        n_eos = eos.numel()
    return B, V, max_new, n_eos


def beam_select(logits: torch.Tensor, step: torch.Tensor, params: torch.Tensor, beam_scores: torch.Tensor,
                history: torch.Tensor, next_ids: torch.Tensor, parent: torch.Tensor, done: torch.Tensor,
                hyp_scores: torch.Tensor, hyp_ids: torch.Tensor, hyp_meta: torch.Tensor, scratch: torch.Tensor,
                num_beams: int, eos: Optional[torch.Tensor] = None, pad_id: int = 0, min_length: int = 0) -> None:
    """One beam-search step in one call (csrc/beam_select_sm100.cu, two kernels): log-softmax, repetition penalty,
    min-length ban and beam score per row, the sequence's top ``max(2, 1 + n_eos) * num_beams`` candidates, then
    ``BeamSearchScorer.process``: new ``beam_scores``, ``next_ids`` and ``parent`` rows, the hypotheses and ``done``
    flags updated in place and ``history`` reordered by parent with the new token appended at column ``step``.
    ``logits`` fp32 (B * num_beams, V); ``step`` (1,) int64 and ``params`` (2,) float64 ``[repetition_penalty,
    length_penalty]`` are read on the device; ``history`` (R, max_new) int64; ``hyp_scores`` (B, num_beams) float64;
    ``hyp_ids`` (B, num_beams, max_new) int64; ``hyp_meta`` (B, num_beams, 2) int64 ``[length (-1 = free), serial]``;
    ``scratch`` >= R * K int64 entries private to the call.  See include/mmfs_b200.h for the rules."""
    B, V, max_new, n_eos = _check_beam_step("beam_select", logits, step, params, 2, beam_scores, history, next_ids,
                                            parent, done, hyp_scores, hyp_ids, hyp_meta, num_beams, eos)
    R = B * num_beams
    _require(scratch.device == logits.device and scratch.dtype == torch.int64 and scratch.is_contiguous()
             and scratch.numel() >= R * beam_candidates(num_beams, n_eos),
             "beam_select: scratch must be contiguous int64 with R * max(2, 1 + n_eos) * num_beams entries")
    with torch.cuda.device(logits.device):
        rc = _lib.lib().mmfs_beam_select(logits.data_ptr(), logits.stride(0), step.data_ptr(), params.data_ptr(),
                                         beam_scores.data_ptr(), history.data_ptr(), next_ids.data_ptr(), parent.data_ptr(),
                                         done.data_ptr(), hyp_scores.data_ptr(), hyp_ids.data_ptr(), hyp_meta.data_ptr(),
                                         eos.data_ptr() if eos is not None else None, n_eos, int(pad_id), int(min_length),
                                         scratch.data_ptr(), B, num_beams, V, max_new, _stream())
    _lib.check(rc, "beam_select")
    launch_counter[0] += 2


def beam_sample_supported(num_beams: int, n_eos: int, V: int) -> bool:
    """Whether ``beam_sample`` takes this shape (its limits: num_beams <= 8, n_eos <= 4, 2 * num_beams <= V <= 2^17)."""
    return (1 <= num_beams <= _lib.BEAM_MAX_BEAMS and 0 <= n_eos <= _lib.BEAM_MAX_EOS
            and 2 * num_beams <= V <= SELECT_MAX_V)


def beam_sample_scratch(num_beams: int, rows: int) -> int:
    """int64 entries of the ``scratch`` of ``beam_sample`` over ``rows`` beam rows: two words per drawn candidate."""
    return rows * 4 * num_beams


def beam_sample(logits: torch.Tensor, step: torch.Tensor, params: torch.Tensor, beam_scores: torch.Tensor,
                history: torch.Tensor, next_ids: torch.Tensor, parent: torch.Tensor, done: torch.Tensor,
                hyp_scores: torch.Tensor, hyp_ids: torch.Tensor, hyp_meta: torch.Tensor, error: torch.Tensor,
                scratch: torch.Tensor, num_beams: int, eos: Optional[torch.Tensor] = None, pad_id: int = 0,
                min_length: int = 0, top_k: int = 50, seed: Optional[torch.Tensor] = None,
                uniforms: Optional[torch.Tensor] = None) -> None:
    """One beam-sample step in one call (csrc/beam_select_sm100.cu, two kernels): ``beam_select``'s row scores, then
    temperature, top-k (``min(max(top_k, 2), V)``; 0 = none) and top-p with two tokens always kept, then 2 * num_beams
    candidates per sequence drawn without replacement from the softmax of the warped scores, ordered by warped score,
    and ``BeamSearchScorer.process`` as in ``beam_select``.  ``params`` (4,) float64 ``[repetition_penalty,
    length_penalty, temperature, top_p]`` and ``seed`` (1,) int64 are read on the device; ``uniforms`` (R, V) fp32 in
    (0, 1) replaces the Philox draw when given; ``error`` (1,) int32 is set to 1 (and stays set) when a sequence gets
    fewer than num_beams non-eos candidates; ``scratch`` >= ``beam_sample_scratch(num_beams, R)`` int64 entries private
    to the call; the other buffers as ``beam_select``.  See include/mmfs_b200.h for the rules."""
    B, V, max_new, n_eos = _check_beam_step("beam_sample", logits, step, params, 4, beam_scores, history, next_ids,
                                            parent, done, hyp_scores, hyp_ids, hyp_meta, num_beams, eos)
    R, dev = B * num_beams, logits.device
    _require(error.device == dev and error.dtype == torch.int32 and error.numel() == 1,
             "beam_sample: error must be a (1,) int32 device tensor")
    _require(scratch.device == dev and scratch.dtype == torch.int64 and scratch.is_contiguous()
             and scratch.numel() >= beam_sample_scratch(num_beams, R),
             "beam_sample: scratch must be contiguous int64 with R * 4 * num_beams entries")
    _require(seed is not None or uniforms is not None, "beam_sample: needs a seed or uniforms")
    if seed is not None:
        _require(seed.device == dev and seed.dtype == torch.int64 and seed.numel() == 1, "beam_sample: seed must be a (1,) int64 device tensor")
    if uniforms is not None:
        _require(uniforms.device == dev and uniforms.dtype == torch.float32 and tuple(uniforms.shape) == (R, V)
                 and uniforms.is_contiguous(), "beam_sample: uniforms must be a contiguous fp32 (R, V) tensor")
    _require(top_k >= 0, "beam_sample: top_k must be >= 0")
    with torch.cuda.device(dev):
        rc = _lib.lib().mmfs_beam_sample(logits.data_ptr(), logits.stride(0), step.data_ptr(), params.data_ptr(),
                                         seed.data_ptr() if seed is not None else None,
                                         uniforms.data_ptr() if uniforms is not None else None, beam_scores.data_ptr(),
                                         history.data_ptr(), next_ids.data_ptr(), parent.data_ptr(), done.data_ptr(),
                                         hyp_scores.data_ptr(), hyp_ids.data_ptr(), hyp_meta.data_ptr(), error.data_ptr(),
                                         eos.data_ptr() if eos is not None else None, n_eos, int(pad_id), int(min_length),
                                         int(top_k), scratch.data_ptr(), B, num_beams, V, max_new, _stream())
    _lib.check(rc, "beam_sample")
    launch_counter[0] += 2


def kv_beam_reorder(kv: torch.Tensor, parent: torch.Tensor, cur: torch.Tensor, step: torch.Tensor, num_beams: int,
                    max_positions: int, done: Optional[torch.Tensor] = None) -> None:
    """Beam search's KV-cache reorder in place, generated positions only, in one launch over every cache tensor:
    ``kv`` (n, R, T_max, ...) holds n caches (every layer's K and V) with dense rows; within each group of
    ``num_beams`` rows, row j takes the contents of row ``parent[j]`` at positions ``[cur - step, cur)``.  ``cur`` and
    ``step`` are (1,) int64 device tensors (``step <= max_positions``); groups with ``done`` set are skipped."""
    inference_only("kv_beam_reorder", kv)
    _require(kv.is_cuda and kv.dim() >= 3, "kv_beam_reorder: kv must be a CUDA (n, R, T_max, ...) tensor")
    n, R, T = kv.shape[:3]
    dev = kv.device
    row_bytes = kv[0, 0, 0].numel() * kv.element_size()
    _require(kv[0, 0, 0].is_contiguous() and kv.stride(2) * kv.element_size() >= row_bytes,
             "kv_beam_reorder: each (cache, row, position) entry must be dense")
    _require(num_beams > 0 and R % num_beams == 0, "kv_beam_reorder: the rows must be whole groups of num_beams")
    _require(parent.device == dev and parent.dtype == torch.int64 and parent.numel() == R and parent.is_contiguous(),
             "kv_beam_reorder: parent must be contiguous int64 with R entries")
    for t, name in ((cur, "cur"), (step, "step")):
        _require(t.device == dev and t.dtype == torch.int64 and t.numel() == 1, f"kv_beam_reorder: {name} must be a (1,) int64 device tensor")
    if done is not None:
        _require(done.device == dev and done.dtype in (torch.bool, torch.uint8) and done.numel() == R // num_beams
                 and done.is_contiguous(), "kv_beam_reorder: done must be contiguous bool / uint8 with one entry per group")
    _require(0 < max_positions <= T, "kv_beam_reorder: max_positions must be in [1, T_max]")
    es = kv.element_size()
    with torch.cuda.device(dev):
        rc = _lib.lib().mmfs_kv_beam_reorder(kv.data_ptr(), n, kv.stride(0) * es, R, kv.stride(1) * es, kv.stride(2) * es,
                                             row_bytes, num_beams, parent.data_ptr(), cur.data_ptr(), step.data_ptr(),
                                             done.data_ptr() if done is not None else None, int(max_positions), _stream())
    _lib.check(rc, "kv_beam_reorder")
    launch_counter[0] += 1


def swiglu(gate_up: torch.Tensor) -> torch.Tensor:
    """act_fn(gate) * up on a (..., 2*I) tensor holding [gate | up] (LlamaMLP, :188-189)."""
    inference_only("swiglu", gate_up)
    _require(gate_up.is_cuda and gate_up.is_contiguous() and gate_up.shape[-1] % 2 == 0, "swiglu: bad input")
    inter = gate_up.shape[-1] // 2
    out = torch.empty(gate_up.shape[:-1] + (inter,), dtype=gate_up.dtype, device=gate_up.device)
    with torch.cuda.device(gate_up.device):
        rc = _lib.lib().mmfs_swiglu(gate_up.data_ptr(), out.data_ptr(), gate_up.numel() // (2 * inter), inter,
                                    _DTYPE_CODE[gate_up.dtype], _stream())
    _lib.check(rc, "swiglu")
    launch_counter[0] += 1
    return out


def geglu(value_gate: torch.Tensor) -> torch.Tensor:
    """value * gelu(gate) (exact erf GELU) on a (..., 2*I) tensor holding [value | gate] (diffusers GEGLU)."""
    inference_only("geglu", value_gate)
    _require(value_gate.is_cuda and value_gate.is_contiguous() and value_gate.shape[-1] % 2 == 0, "geglu: bad input")
    inter = value_gate.shape[-1] // 2
    out = torch.empty(value_gate.shape[:-1] + (inter,), dtype=value_gate.dtype, device=value_gate.device)
    with torch.cuda.device(value_gate.device):
        rc = _lib.lib().mmfs_geglu(value_gate.data_ptr(), out.data_ptr(), value_gate.numel() // (2 * inter), inter,
                                   _DTYPE_CODE[value_gate.dtype], _stream())
    _lib.check(rc, "geglu")
    launch_counter[0] += 1
    return out


def attention(q, k, v, key_mask=None, causal=True, past=0, scale=None, force_generic=False) -> torch.Tensor:
    """softmax(q k^T * scale + mask) v.  q (B,Tq,H,hd), k/v (B,Tkv,H,hd) -- any batch / token strides, heads
    dense; key_mask (B,Tkv) bool/uint8 (1 = attend) or None; causal: query i sees keys j <= past + i.
    Returns (B, Tq, H*hd).  Prefill shapes go to the wgmma kernel, decode / odd shapes to the
    bandwidth kernel (see csrc/attn_generic_sm100.cu)."""
    B, Tq, H, hd = q.shape
    Tkv = k.shape[1]
    for t in (q, k, v):
        _require(t.is_cuda and t.stride(3) == 1 and t.stride(2) == hd, "attention: heads must be dense (.., H, hd)")
    inference_only("attention", q, k, v)
    _require(k.shape == v.shape and k.shape[0] == B and k.shape[2] == H and k.shape[3] == hd, "attention: k/v shape mismatch")
    scale = float(scale if scale is not None else hd ** -0.5)
    out = torch.empty((B, Tq, H, hd), dtype=q.dtype, device=q.device)
    km = None
    if key_mask is not None:
        km = key_mask.to(torch.uint8).contiguous()
        _require(tuple(km.shape) == (B, Tkv), "attention: key_mask must be (B, Tkv)")
    from . import attn_tc
    es = q.element_size()
    decode_ok = (Tq == 1 and not force_generic and q.dtype != torch.float64 and hd % 32 == 0 and hd <= 256 and
                 (hd * es) % 16 == 0 and all(t.data_ptr() % 16 == 0 and (t.stride(0) * es) % 16 == 0 and
                                            (t.stride(1) * es) % 16 == 0 for t in (k, v)))
    if not force_generic and attn_tc.supported(q, k, v, Tq, Tkv, hd):
        attn_tc.forward(q, k, v, out, km, causal, past, scale)
    elif decode_ok:      # one query row over a KV cache: split-KV kernel (K and V read once, all SMs busy)
        lib = _lib.lib()
        scratch = torch.empty((lib.mmfs_attn_decode_scratch_floats(B, H, Tkv, hd),), dtype=torch.float32, device=q.device)
        with torch.cuda.device(q.device):
            rc = lib.mmfs_attn_decode(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(),
                                      km.data_ptr() if km is not None else None, scratch.data_ptr(), B, H, Tkv, hd,
                                      q.stride(0), k.stride(0), k.stride(1), v.stride(0), v.stride(1), out.stride(0), scale,
                                      1 if causal else 0, int(past), _DTYPE_CODE[q.dtype], _stream())
        _lib.check(rc, "attention (decode)")
        launch_counter[0] += 1
    else:
        with torch.cuda.device(q.device):
            rc = _lib.lib().mmfs_attn_generic(
                q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), km.data_ptr() if km is not None else None,
                B, H, Tq, Tkv, hd, q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1),
                out.stride(0), out.stride(1), scale, 1 if causal else 0, int(past), _DTYPE_CODE[q.dtype], _stream())
        _lib.check(rc, "attention")
    launch_counter[0] += 1
    return out.view(B, Tq, H * hd)


# ---- training path: backward kernels (csrc/attn_bwd_sm100.cu, csrc/llama_ops_sm100.cu).  autograd_ops.py wraps them in
# autograd Functions; like the forward wrappers they refuse to run where autograd would record them.

def _check_qkv_view(t, B, T, H, hd, what):
    _require(t.is_cuda and tuple(t.shape) == (B, T, H, hd) and t.stride(3) == 1 and t.stride(2) == hd,
             f"{what}: tensors must be (B, T, H, hd) CUDA views with dense heads")


def attention_forward_lse(q, k, v, key_mask=None, scale=None, causal=True):
    """``attention`` on the wgmma kernel that also returns the row log-sum-exp: ``(out (B,Tq,H,hd), lse (B,H,Tq)
    fp32)``, natural log, +inf for a row that sees no key.  ``out`` is bit-identical to ``attention``'s on the same
    kernel.  q (B,Tq,H,hd), k / v (B,Tkv,H,hd); causal needs Tq = Tkv (query i sees keys j <= i)."""
    B, Tq, H, hd = q.shape
    Tkv = k.shape[1]
    inference_only("attention_forward_lse", q, k, v)
    _check_qkv_view(q, B, Tq, H, hd, "attention_forward_lse")
    for t in (k, v):
        _check_qkv_view(t, B, Tkv, H, hd, "attention_forward_lse")
    _require(not causal or Tq == Tkv, "attention_forward_lse: causal attention needs Tq == Tkv")
    scale = float(scale if scale is not None else hd ** -0.5)
    out = torch.empty((B, Tq, H, hd), dtype=q.dtype, device=q.device)
    lse = torch.empty((B, H, Tq), dtype=torch.float32, device=q.device)
    km = None
    if key_mask is not None:
        km = key_mask.to(torch.uint8).contiguous()
        _require(tuple(km.shape) == (B, Tkv), "attention_forward_lse: key_mask must be (B, Tkv)")
    counter = torch.empty((1,), dtype=torch.int32, device=q.device)
    with torch.cuda.device(q.device):
        rc = _lib.lib().mmfs_attn_forward_lse(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), km.data_ptr() if km is not None else None,
            B, H, Tq, Tkv, hd, q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1),
            out.stride(0), out.stride(1), scale, 1 if causal else 0, 0, _DTYPE_CODE[q.dtype], counter.data_ptr(), _stream())
    _lib.check(rc, "attention_forward_lse")
    launch_counter[0] += 1
    return out, lse


def attention_backward(q, k, v, out, d_out, lse, dq, dk, dv, key_mask=None, scale=None) -> None:
    """dQ, dK, dV of causal ``attention_forward_lse`` (hd 128, bf16 / fp16), written into the (B, T, H, hd) views
    ``dq`` / ``dk`` / ``dv`` -- e.g. slices of one (B, T, 3, H, hd) buffer, so that the QKV projection's backward is
    one GEMM.  Deterministic: no atomics, two calls give bit-identical results."""
    B, T, H, hd = q.shape
    inference_only("attention_backward", q, k, v, out, d_out)
    for t in (q, k, v, out, d_out, dq, dk, dv):
        _check_qkv_view(t, B, T, H, hd, "attention_backward")
    _require(all(t.dtype == q.dtype for t in (k, v, out, d_out, dq, dk, dv)), "attention_backward: dtype mismatch")
    _require(lse.dtype == torch.float32 and tuple(lse.shape) == (B, H, T) and lse.is_contiguous(),
             "attention_backward: lse must be contiguous fp32 (B, H, T)")
    scale = float(scale if scale is not None else hd ** -0.5)
    km = None
    if key_mask is not None:
        km = key_mask.to(torch.uint8).contiguous()
        _require(tuple(km.shape) == (B, T), "attention_backward: key_mask must be (B, T)")
    delta = torch.empty((B, H, T), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        rc = _lib.lib().mmfs_attn_backward(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), d_out.data_ptr(), lse.data_ptr(), dq.data_ptr(),
            dk.data_ptr(), dv.data_ptr(), delta.data_ptr(), km.data_ptr() if km is not None else None, B, H, T, hd,
            q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1), out.stride(0), out.stride(1),
            d_out.stride(0), d_out.stride(1), dq.stride(0), dq.stride(1), dk.stride(0), dk.stride(1), dv.stride(0),
            dv.stride(1), scale, _DTYPE_CODE[q.dtype], _stream())
    _lib.check(rc, "attention_backward")
    launch_counter[0] += 3


def attention_backward_general(q, k, v, out, d_out, lse, dq, dk, dv, key_mask=None, scale=None, causal=False) -> None:
    """dQ, dK, dV of ``attention_forward_lse`` for q / out / d_out / dq (B, Tq, H, hd) and k / v / dk / dv (B, Tkv, H, hd)
    views, hd 64 or 128, bf16 / fp16, causal (Tq = Tkv) or not, ``key_mask`` (B, Tkv) or None.  Same kernels and
    determinism as ``attention_backward``."""
    B, Tq, H, hd = q.shape
    Tkv = k.shape[1]
    inference_only("attention_backward_general", q, k, v, out, d_out)
    for t in (q, out, d_out, dq):
        _check_qkv_view(t, B, Tq, H, hd, "attention_backward_general")
    for t in (k, v, dk, dv):
        _check_qkv_view(t, B, Tkv, H, hd, "attention_backward_general")
    _require(all(t.dtype == q.dtype for t in (k, v, out, d_out, dq, dk, dv)), "attention_backward_general: dtype mismatch")
    _require(lse.dtype == torch.float32 and tuple(lse.shape) == (B, H, Tq) and lse.is_contiguous(),
             "attention_backward_general: lse must be contiguous fp32 (B, H, Tq)")
    scale = float(scale if scale is not None else hd ** -0.5)
    km = None
    if key_mask is not None:
        km = key_mask.to(torch.uint8).contiguous()
        _require(tuple(km.shape) == (B, Tkv), "attention_backward_general: key_mask must be (B, Tkv)")
    delta = torch.empty((B, H, Tq), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        rc = _lib.lib().mmfs_attn_backward_general(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), d_out.data_ptr(), lse.data_ptr(), dq.data_ptr(),
            dk.data_ptr(), dv.data_ptr(), delta.data_ptr(), km.data_ptr() if km is not None else None, B, H, Tq, Tkv, hd,
            q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1), out.stride(0), out.stride(1),
            d_out.stride(0), d_out.stride(1), dq.stride(0), dq.stride(1), dk.stride(0), dk.stride(1), dv.stride(0),
            dv.stride(1), scale, 1 if causal else 0, _DTYPE_CODE[q.dtype], _stream())
    _lib.check(rc, "attention_backward_general")
    launch_counter[0] += 3


def rmsnorm_backward(x: torch.Tensor, weight: torch.Tensor, dy: torch.Tensor, eps: float, weight_grad: bool = True):
    """(dx, dweight) of ``rmsnorm`` over the last dim; dweight is None unless ``weight_grad``.  dweight is reduced from
    fixed per-CTA partials in a fixed order (run-to-run reproducible)."""
    inference_only("rmsnorm_backward", x, weight, dy)
    _require(x.is_cuda and x.is_contiguous() and dy.is_contiguous() and weight.is_contiguous() and dy.shape == x.shape,
             "rmsnorm_backward: contiguous CUDA tensors of one shape required")
    _require(weight.dtype == x.dtype == dy.dtype and weight.numel() == x.shape[-1], "rmsnorm_backward: weight dtype / size mismatch")
    cols = x.shape[-1]
    rows = x.numel() // cols
    dx = torch.empty_like(x)
    dw = torch.empty_like(weight) if weight_grad else None
    partials = (torch.empty((min(rows, _lib.RMSNORM_BWD_PARTS), cols), dtype=torch.float32, device=x.device)
                if weight_grad else None)
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_rmsnorm_backward(x.data_ptr(), weight.data_ptr(), dy.data_ptr(), dx.data_ptr(),
                                              dw.data_ptr() if dw is not None else None,
                                              partials.data_ptr() if partials is not None else None, rows, cols, float(eps),
                                              _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "rmsnorm_backward")
    launch_counter[0] += 2 if weight_grad else 1
    return dx, dw


def layernorm_backward(x: torch.Tensor, weight: torch.Tensor, dy: torch.Tensor, eps: float, weight_grad: bool = True,
                       bias_grad: bool = True):
    """(dx, dweight, dbias) of ``layernorm`` over the last dim, statistics recomputed from x in fp32; dweight / dbias
    are None unless asked for.  They are reduced from fixed per-CTA partials in a fixed order (run-to-run
    reproducible)."""
    inference_only("layernorm_backward", x, weight, dy)
    _require(x.is_cuda and x.is_contiguous() and dy.is_contiguous() and weight.is_contiguous() and dy.shape == x.shape,
             "layernorm_backward: contiguous CUDA tensors of one shape required")
    _require(weight.dtype == x.dtype == dy.dtype and weight.numel() == x.shape[-1],
             "layernorm_backward: weight dtype / size mismatch")
    cols = x.shape[-1]
    rows = x.numel() // cols
    dx = torch.empty_like(x)
    dw = torch.empty_like(weight) if weight_grad else None
    db = torch.empty_like(weight) if bias_grad else None
    partials = (torch.empty((2, min(rows, _lib.RMSNORM_BWD_PARTS), cols), dtype=torch.float32, device=x.device)
                if weight_grad or bias_grad else None)
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_layernorm_backward(x.data_ptr(), weight.data_ptr(), dy.data_ptr(), dx.data_ptr(),
                                                dw.data_ptr() if dw is not None else None,
                                                db.data_ptr() if db is not None else None,
                                                partials.data_ptr() if partials is not None else None, rows, cols,
                                                float(eps), _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "layernorm_backward")
    launch_counter[0] += 2 if partials is not None else 1
    return dx, dw, db


def swiglu_backward(gate_up: torch.Tensor, d_out: torch.Tensor) -> torch.Tensor:
    """d(gate_up) of ``swiglu``: [d gate | d up], computed in fp32."""
    inference_only("swiglu_backward", gate_up, d_out)
    _require(gate_up.is_cuda and gate_up.is_contiguous() and d_out.is_contiguous() and gate_up.shape[-1] % 2 == 0
             and d_out.shape == gate_up.shape[:-1] + (gate_up.shape[-1] // 2,) and d_out.dtype == gate_up.dtype,
             "swiglu_backward: bad input")
    inter = gate_up.shape[-1] // 2
    d_gu = torch.empty_like(gate_up)
    with torch.cuda.device(gate_up.device):
        rc = _lib.lib().mmfs_swiglu_backward(gate_up.data_ptr(), d_out.data_ptr(), d_gu.data_ptr(),
                                             gate_up.numel() // (2 * inter), inter, _DTYPE_CODE[gate_up.dtype], _stream())
    _lib.check(rc, "swiglu_backward")
    launch_counter[0] += 1
    return d_gu


def geglu_backward(value_gate: torch.Tensor, d_out: torch.Tensor) -> torch.Tensor:
    """d(value_gate) of ``geglu``: [d value | d gate], computed in fp32 and rounded once."""
    inference_only("geglu_backward", value_gate, d_out)
    _require(value_gate.is_cuda and value_gate.is_contiguous() and d_out.is_contiguous() and value_gate.shape[-1] % 2 == 0
             and d_out.shape == value_gate.shape[:-1] + (value_gate.shape[-1] // 2,) and d_out.dtype == value_gate.dtype
             and d_out.device == value_gate.device, "geglu_backward: bad input")
    inter = value_gate.shape[-1] // 2
    d_vg = torch.empty_like(value_gate)
    with torch.cuda.device(value_gate.device):
        rc = _lib.lib().mmfs_geglu_backward(value_gate.data_ptr(), d_out.data_ptr(), d_vg.data_ptr(),
                                            value_gate.numel() // (2 * inter), inter, _DTYPE_CODE[value_gate.dtype], _stream())
    _lib.check(rc, "geglu_backward")
    launch_counter[0] += 1
    return d_vg


def quick_gelu_backward(h: torch.Tensor, dy: torch.Tensor) -> torch.Tensor:
    """dh of CLIP's quick_gelu ``h * sigmoid(1.702 h)``, computed in fp32 and rounded once (csrc/vit_bwd_sm100.cu)."""
    inference_only("quick_gelu_backward", h, dy)
    _require(h.is_cuda and h.is_contiguous() and dy.is_contiguous() and dy.shape == h.shape and dy.dtype == h.dtype,
             "quick_gelu_backward: contiguous CUDA tensors of one shape and dtype required")
    dh = torch.empty_like(h)
    with torch.cuda.device(h.device):
        rc = _lib.lib().mmfs_quick_gelu_backward(h.data_ptr(), dy.data_ptr(), dh.data_ptr(), h.numel(),
                                                 _DTYPE_CODE[h.dtype], _stream())
    _lib.check(rc, "quick_gelu_backward")
    launch_counter[0] += 1
    return dh


def image_reentry(images: torch.Tensor, size: int = 224, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """A generated (N, 3, S, S) fp32 image in [0, 1] as the visual tokenizer's (N, 3, size, size) fp32 input, on the
    device and bit-identical to the reference's host path (``tensor_to_pil``, ``center_crop_arr``, ``/ 255``; see
    csrc/image_reentry_sm100.cu).  ``out`` (contiguous, e.g. a slot of the sample's image tensor) receives the result.
    Non-square or non-RGB images raise."""
    _require(images.is_cuda and images.dim() == 4 and images.dtype == torch.float32,
             "image_reentry: images must be a (N, 3, S, S) fp32 CUDA tensor")
    images = images.contiguous()
    N, C, H, W = images.shape
    if out is None:
        out = torch.empty((N, C, size, size), dtype=torch.float32, device=images.device)
    _require(out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and out.device == images.device and
             tuple(out.shape) == (N, C, size, size), "image_reentry: out must be a contiguous (N, 3, size, size) fp32 "
             "tensor on the images' device")
    with torch.cuda.device(images.device):
        rc = _lib.lib().mmfs_image_reentry(images.data_ptr(), out.data_ptr(), N, C, H, W, int(size), _stream())
    _lib.check(rc, "image_reentry")
    launch_counter[0] += 1
    return out


def _pixel_stride(t: torch.Tensor):
    """The one stride that steps pixel p = y * W + x of a (B, C, H, W) tensor, or None when H and W are not laid out
    as one flattened pixel axis.  The stride of a size-1 dim is arbitrary in PyTorch and is not used."""
    H, W = t.shape[2:]
    if W > 1:
        return t.stride(3) if H == 1 or t.stride(2) == W * t.stride(3) else None
    return t.stride(2) if H > 1 else 1


def resize_bilinear_backward(dy: torch.Tensor, in_hw, scale_factor: float) -> torch.Tensor:
    """dx of ``F.interpolate(x, scale_factor=scale_factor, mode="bilinear", align_corners=False)`` for an x of spatial
    size ``in_hw`` and the (B, C, Hout, Wout) gradient ``dy`` (read through its strides; NCHW and the token layout
    (B, Hout*Wout, C) viewed as NCHW need no copy).  Returns dx in the token layout (B, Hin*Win, C), contiguous.
    Gather form without atomics: bit-reproducible."""
    inference_only("resize_bilinear_backward", dy)
    Hin, Win = int(in_hw[0]), int(in_hw[1])
    _require(dy.is_cuda and dy.dim() == 4, "resize_bilinear_backward: dy must be a (B, C, Hout, Wout) CUDA tensor")
    B, C, Hout, Wout = dy.shape
    _require((Hout, Wout) == (math.floor(Hin * scale_factor), math.floor(Win * scale_factor)),
             "resize_bilinear_backward: dy's size is not the input size times the scale factor")
    ps = _pixel_stride(dy)
    if ps is None:
        dy = dy.contiguous()
        ps = _pixel_stride(dy)
    dx = torch.empty((B, Hin * Win, C), dtype=dy.dtype, device=dy.device)
    scale = float(1.0 / scale_factor)
    with torch.cuda.device(dy.device):
        rc = _lib.lib().mmfs_resize_bilinear_backward(dy.data_ptr(), dx.data_ptr(), B, C, Hin, Win, Hout, Wout, dy.stride(0),
                                                      dy.stride(1), ps, scale, scale, _DTYPE_CODE[dy.dtype], _stream())
    _lib.check(rc, "resize_bilinear_backward")
    launch_counter[0] += 1
    return dx


def conv2d_supported(x: torch.Tensor, weight: torch.Tensor, stride: int, padding: int) -> bool:
    """Whether ``conv2d`` can take this layer (else the caller keeps it on cuDNN: conv_in / conv_out of the UNet)."""
    if x.dtype not in (torch.bfloat16, torch.float16) or not x.is_cuda or x.dim() != 4:
        return False
    B, Cin, H, W = x.shape
    Cout, _, KH, KW = weight.shape
    Ho, Wo = (H + 2 * padding - KH) // stride + 1, (W + 2 * padding - KW) // stride + 1
    tile = (Wo % 16 == 0 and Ho % 8 == 0) or (Wo == 8 and Ho == 8 and B % 2 == 0)
    return Cin % 64 == 0 and (Cout % 160 == 0 or Cout % 128 == 0) and stride in (1, 2) and tile


def conv2d(x: torch.Tensor, weight_khwc: torch.Tensor, bias=None, stride: int = 1, padding: int = 0, add_bc=None,
           residual=None) -> torch.Tensor:
    """Implicit-GEMM convolution on the tensor cores (csrc/conv_igemm_sm100.cu).  ``x`` is a (B, Cin, H, W) tensor in
    channels_last memory format (i.e. NHWC in memory); ``weight_khwc`` is the filter permuted to (Cout, KH, KW, Cin),
    contiguous; returns (B, Cout, Ho, Wo) channels_last.  Optional fused epilogue: ``bias`` (Cout), ``add_bc``
    (B, Cout) broadcast over pixels, ``residual`` (like the output, channels_last)."""
    B, Cin, H, W = x.shape
    Cout, KH, KW, _ = weight_khwc.shape
    inference_only("conv2d", x, weight_khwc, bias, add_bc, residual)
    _require(x.is_contiguous(memory_format=torch.channels_last) and weight_khwc.is_contiguous(), "conv2d: x must be channels_last")
    Ho, Wo = (H + 2 * padding - KH) // stride + 1, (W + 2 * padding - KW) // stride + 1
    out = torch.empty((B, Cout, Ho, Wo), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    if residual is not None:
        _require(residual.shape == out.shape and residual.is_contiguous(memory_format=torch.channels_last), "conv2d: residual layout")
    if add_bc is not None:
        add_bc = add_bc.contiguous()
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_conv2d_nhwc(
            x.data_ptr(), weight_khwc.data_ptr(), bias.data_ptr() if bias is not None else None,
            add_bc.data_ptr() if add_bc is not None else None, residual.data_ptr() if residual is not None else None,
            out.data_ptr(), B, H, W, Cin, Cout, KH, KW, stride, padding, _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "conv2d")
    launch_counter[0] += 1
    return out


def fold_up2x_weights(weight: torch.Tensor) -> torch.Tensor:
    """A 3x3 filter (Cout, Cin, 3, 3) folded for ``conv2d_up2x``: (4, Cout, 2, 2, Cin), phase p = 2 py + px.

    ``conv3x3(up2x(x), pad 1)`` at output pixel (2i + py, 2j + px) reads the low-resolution rows {i-1, i, i} (py = 0)
    or {i, i, i+1} (py = 1), so along rows the taps fold to {w0, w1 + w2} at offsets {-1, 0} or {w0 + w1, w2} at
    {0, +1}, and the same along columns.  Summed in fp32 (fp64 stays fp64) and rounded to the filter's dtype once."""
    acc = torch.float64 if weight.dtype == torch.float64 else torch.float32
    fold = torch.tensor([[[1, 0, 0], [0, 1, 1]], [[1, 1, 0], [0, 0, 1]]], dtype=acc, device=weight.device)   # (py, tap, k)
    w = torch.einsum("pak,ockl,qbl->pqoabc", fold, weight.to(acc), fold)         # (py, px, Cout, 2, 2, Cin)
    return w.reshape(4, *w.shape[2:]).to(weight.dtype).contiguous()


def dgrad_weights_khwc(weight: torch.Tensor) -> torch.Tensor:
    """The filter of the data gradient of a stride-1, 'same'-padded convolution, in ``conv2d``'s KHWC layout.

    For y = conv(x, W) with a KxK filter and pad (K-1)/2, dx = conv(dy, W') with the same padding, where W' swaps the
    channel roles and rotates the taps by 180 degrees: ``W'[ci, ky, kx, co] = W[co, ci, K-1-ky, K-1-kx]``.  A pure
    re-indexing, so no rounding."""
    return weight.flip(2, 3).permute(1, 2, 3, 0).contiguous()


def fold_dgrad_down2x_weights(weight: torch.Tensor) -> torch.Tensor:
    """A 3x3 / stride-2 / pad-1 filter (Cout, Cin, 3, 3) folded into the data gradient's phase filters for ``conv2d_up2x``:
    (4, Cin, 2, 2, Cout), phase p = 2 py + px.

    y[i] = sum_k w[k] x[2i + k - 1] along each axis, so dx at input row 2j (py = 0) is w[1] dy[j], and at row 2j + 1
    (py = 1) w[2] dy[j] + w[0] dy[j + 1]: in ``conv2d_up2x``'s tap order (offsets {-1, 0} for py = 0, {0, +1} for py = 1)
    the rows fold to {0, w1} or {w2, w0}, the columns alike, and the channels are transposed.  Summed in fp32 (fp64 stays
    fp64) and rounded to the filter's dtype once (each tap is a single weight, so the fold is exact)."""
    acc = torch.float64 if weight.dtype == torch.float64 else torch.float32
    fold = torch.tensor([[[0, 0, 0], [0, 1, 0]], [[0, 0, 1], [1, 0, 0]]], dtype=acc, device=weight.device)   # (py, tap, k)
    w = torch.einsum("pak,ockl,qbl->pqcabo", fold, weight.to(acc), fold)         # (py, px, Cin, 2, 2, Cout)
    return w.reshape(4, *w.shape[2:]).to(weight.dtype).contiguous()


def conv2d_up2x_supported(x: torch.Tensor, weight: torch.Tensor) -> bool:
    """Whether ``conv2d_up2x`` can take ``conv3x3(interpolate(x, 2, "nearest"))`` for this (B, Cin, H, W) input and
    (Cout, Cin, 3, 3) filter."""
    if x.dtype not in (torch.bfloat16, torch.float16) or not x.is_cuda or x.dim() != 4 or tuple(weight.shape[2:]) != (3, 3):
        return False
    B, Cin, H, W = x.shape
    Cout = weight.shape[0]
    tile = (W % 16 == 0 and H % 8 == 0) or (W == 8 and H == 8 and B % 2 == 0)
    return Cin % 64 == 0 and (Cout % 160 == 0 or Cout % 128 == 0) and tile


def conv2d_up2x(x: torch.Tensor, weight_phases: torch.Tensor, bias=None) -> torch.Tensor:
    """Nearest 2x upsample + 3x3 / pad-1 convolution in one kernel (csrc/conv_igemm_sm100.cu, phase form): four 2x2
    convolutions over the low-resolution input, the 4x-size upsampled tensor is never formed.  ``x`` (B, Cin, H, W)
    channels_last; ``weight_phases`` from ``fold_up2x_weights``; returns (B, Cout, 2H, 2W) channels_last."""
    B, Cin, H, W = x.shape
    Cout = weight_phases.shape[1]
    inference_only("conv2d_up2x", x, weight_phases, bias)
    _require(x.is_contiguous(memory_format=torch.channels_last) and weight_phases.is_contiguous(), "conv2d_up2x: x must be channels_last")
    _require(tuple(weight_phases.shape) == (4, Cout, 2, 2, Cin), "conv2d_up2x: weights must be (4, Cout, 2, 2, Cin)")
    out = torch.empty((B, Cout, 2 * H, 2 * W), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_conv2d_up2x_nhwc(x.data_ptr(), weight_phases.data_ptr(), bias.data_ptr() if bias is not None else None,
                                              out.data_ptr(), B, H, W, Cin, Cout, _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "conv2d_up2x")
    launch_counter[0] += 1
    return out


def conv2d_down2x_supported(x: torch.Tensor, weight: torch.Tensor) -> bool:
    """Whether ``conv2d_down2x`` can take ``conv3x3(F.pad(x, (0, 1, 0, 1)), stride 2)`` for this (B, Cin, H, W) input and
    (Cout, Cin, 3, 3) filter."""
    if x.dtype not in (torch.bfloat16, torch.float16) or not x.is_cuda or x.dim() != 4 or tuple(weight.shape[2:]) != (3, 3):
        return False
    B, Cin, H, W = x.shape
    Cout = weight.shape[0]
    if H % 2 or W % 2:
        return False
    Ho, Wo = H // 2, W // 2
    tile = (Wo % 16 == 0 and Ho % 8 == 0) or (Wo == 8 and Ho == 8 and B % 2 == 0)
    return Cin % 64 == 0 and (Cout % 160 == 0 or Cout % 128 == 0) and tile


def conv2d_down2x(x: torch.Tensor, weight_khwc: torch.Tensor, bias=None) -> torch.Tensor:
    """diffusers' ``Downsample2D(padding=0)`` -- one zero row at the bottom and one zero column at the right, then a 3x3 /
    stride-2 convolution -- in the implicit-GEMM kernel (csrc/conv_igemm_sm100.cu), the padded copy never formed.  ``x``
    (B, Cin, H, W) channels_last with H, W even; ``weight_khwc`` (Cout, 3, 3, Cin) contiguous; returns (B, Cout, H/2, W/2)
    channels_last."""
    B, Cin, H, W = x.shape
    Cout = weight_khwc.shape[0]
    inference_only("conv2d_down2x", x, weight_khwc, bias)
    _require(x.is_contiguous(memory_format=torch.channels_last) and weight_khwc.is_contiguous(), "conv2d_down2x: x must be channels_last")
    _require(tuple(weight_khwc.shape) == (Cout, 3, 3, Cin), "conv2d_down2x: weights must be (Cout, 3, 3, Cin)")
    out = torch.empty((B, Cout, H // 2, W // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_conv2d_down2x_nhwc(x.data_ptr(), weight_khwc.data_ptr(), bias.data_ptr() if bias is not None else None,
                                                out.data_ptr(), B, H, W, Cin, Cout, _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "conv2d_down2x")
    launch_counter[0] += 1
    return out


def group_norm_supported(x: torch.Tensor) -> bool:
    if not x.is_cuda or x.dim() != 4 or x.dtype not in _DTYPE_CODE or x.dtype == torch.float64:
        return False
    vec = 16 // x.element_size()
    return x.shape[1] % vec == 0 and x.shape[1] // vec <= 1024 and x.is_contiguous(memory_format=torch.channels_last)


def group_norm_nhwc(x: torch.Tensor, groups: int, weight=None, bias=None, eps: float = 1e-5, silu: bool = False) -> torch.Tensor:
    """``F.group_norm`` (+ ``F.silu`` when ``silu``) on a channels_last (B, C, H, W) tensor, result channels_last
    (torch's CUDA group_norm returns NCHW, which costs a layout round trip around each convolution)."""
    inference_only("group_norm_nhwc", x, weight, bias)
    _require(group_norm_supported(x), "group_norm_nhwc: need a CUDA channels_last f32/f16/bf16 tensor with C % (16/size) == 0")
    B, C, H, W = x.shape
    _require(groups > 0 and C % groups == 0, f"group_norm_nhwc: {C} channels do not split into {groups} groups")
    _check_affine("group_norm_nhwc", x, C, weight, bias)
    y = torch.empty_like(x, memory_format=torch.channels_last)
    stats = torch.empty((B, 64, groups, 2), dtype=torch.float32, device=x.device)   # per-chunk (mean, M2) of each group
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_groupnorm_nhwc(x.data_ptr(), weight.data_ptr() if weight is not None else None,
                                            bias.data_ptr() if bias is not None else None, y.data_ptr(), stats.data_ptr(),
                                            B, H * W, C, groups, float(eps), int(silu), _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "group_norm_nhwc")
    launch_counter[0] += 2
    return y


def group_norm_nhwc_backward(x: torch.Tensor, dy: torch.Tensor, groups: int, weight=None, bias=None, eps: float = 1e-5,
                             silu: bool = False) -> torch.Tensor:
    """dx of ``group_norm_nhwc`` (csrc/groupnorm_nhwc_sm100.cu, three kernels): the statistics recomputed from x as the
    forward computes them, the SiLU derivative taken at the forward's rounded pre-activation, every sum reduced in a
    fixed order (run-to-run reproducible).  The affine parameters get no gradient.  ``x`` and ``dy`` channels_last
    (B, C, H, W) of one dtype; returns dx channels_last."""
    inference_only("group_norm_nhwc_backward", x, dy, weight, bias)
    _require(group_norm_supported(x) and x.shape[1] * x.element_size() <= 8192,
             "group_norm_nhwc_backward: need a CUDA channels_last f32/f16/bf16 tensor with C % (16/size) == 0 and "
             "C * size <= 8 KiB")
    _require(dy.shape == x.shape and dy.dtype == x.dtype and dy.device == x.device,
             "group_norm_nhwc_backward: dy must match x in shape, dtype and device")
    if not dy.is_contiguous(memory_format=torch.channels_last):
        dy = dy.contiguous(memory_format=torch.channels_last)
    B, C, H, W = x.shape
    _require(groups > 0 and C % groups == 0, f"group_norm_nhwc_backward: {C} channels do not split into {groups} groups")
    _check_affine("group_norm_nhwc_backward", x, C, weight, bias)
    dx = torch.empty_like(x, memory_format=torch.channels_last)
    scratch = torch.empty((2, B, 64, groups, 2), dtype=torch.float32, device=x.device)   # statistics, then (sum g, sum g xhat)
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_groupnorm_nhwc_backward(x.data_ptr(), weight.data_ptr() if weight is not None else None,
                                                     bias.data_ptr() if bias is not None else None, dy.data_ptr(),
                                                     dx.data_ptr(), scratch.data_ptr(), B, H * W, C, groups, float(eps),
                                                     int(silu), _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "group_norm_nhwc_backward")
    launch_counter[0] += 3
    return dx
