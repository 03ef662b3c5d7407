"""Tensor-level wrappers of the decoder-layer kernels (csrc/llama_ops_sm100.cu, csrc/attn_*.cu).

Host side is PyTorch (allocation, streams); every function enqueues exactly one hand-written kernel
through the C ABI and raises if the library rejects the arguments -- there is no PyTorch fallback.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib
from .msda import _DTYPE_CODE, _require

launch_counter = [0]   # kernels of ours launched through this module (bench.py's gpu_launches)


def inference_only(name: str, *tensors) -> None:
    """None of the ctypes kernels is autograd-aware: refuse to run where a gradient would be silently dropped."""
    if torch.is_grad_enabled() and any(t is not None and torch.is_tensor(t) and t.requires_grad for t in tensors):
        raise RuntimeError(f"{name}: this kernel is inference-only (no autograd support); call it under torch.no_grad() "
                           "or detach its inputs / freeze its parameters")


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


def layernorm(x: torch.Tensor, weight, bias, eps: float) -> torch.Tensor:
    inference_only("layernorm", x, weight, bias)
    _require(x.is_cuda and x.is_contiguous(), "layernorm: contiguous CUDA tensor required")
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


_SKINNY_SCRATCH = {}   # device -> zeroed fp32 scratch (tickets + partial tiles), shared by every call on the device


def linear_skinny_shape_ok(M: int, N: int, K: int) -> bool:
    """At most 8 rows, N % 32 == 0, K % 512 == 0, the x rows + at least two 32 KB stages of the copy ring inside shared
    memory (``csrc/linear_skinny_sm100.cu``): 8 rows up to K = 9216, 4 rows up to K = 18432."""
    return (1 <= M <= 8 and N % 32 == 0 and N <= 32 << 16 and K % 512 == 0 and
            2 * 32768 + M * (K * 2 + 64) + 16912 <= 227 * 1024)


def linear_skinny_supported(x: torch.Tensor, weight: torch.Tensor, prologue: int = 0) -> bool:
    """Whether ``linear_skinny`` takes this call: CUDA, f16 / bf16, contiguous, ``linear_skinny_shape_ok``."""
    N, K = weight.shape
    M = x.numel() // (K * (2 if prologue == 2 else 1))
    return (x.is_cuda and x.dtype in (torch.float16, torch.bfloat16) and weight.dtype == x.dtype and x.is_contiguous()
            and weight.is_contiguous() and linear_skinny_shape_ok(M, N, K))


def linear_skinny(x: torch.Tensor, weight: torch.Tensor, residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                  norm_weight: Optional[torch.Tensor] = None, eps: float = 0.0, swiglu: bool = False) -> torch.Tensor:
    """Decode-step linear ``prologue(x) @ weight^T (+ residual)`` for at most 8 rows (see ``mmfs_linear_skinny`` in
    include/mmfs_b200.h).  ``norm_weight``: fold LlamaRMSNorm(x) in front; ``swiglu``: x is ``[gate | up]`` rows of
    2K columns and the operand is silu(gate) * up.  ``out`` may be ``residual`` itself (in-place residual stream)."""
    prologue = 1 if norm_weight is not None else (2 if swiglu else 0)
    N, K = weight.shape
    M = x.numel() // (K * (2 if swiglu else 1))
    _require(linear_skinny_supported(x, weight, prologue), "linear_skinny: unsupported shape / dtype (see linear_skinny_supported)")
    inference_only("linear_skinny", x, weight)
    if out is None:
        out = torch.empty(tuple(x.shape[:-1]) + (N,), dtype=x.dtype, device=x.device)
    _require(out.is_contiguous() and out.numel() == M * N and out.dtype == x.dtype, "linear_skinny: out must be contiguous (M, N)")
    if residual is not None:
        _require(residual.is_contiguous() and residual.numel() == M * N and residual.dtype == x.dtype,
                 "linear_skinny: residual must be contiguous (M, N)")
    if norm_weight is not None:
        _require(norm_weight.is_contiguous() and norm_weight.numel() == K and norm_weight.dtype == x.dtype,
                 "linear_skinny: norm_weight must be (K,) in x.dtype")
    lib = _lib.lib()
    need = lib.mmfs_linear_skinny_scratch_floats(N)
    key = (x.device.type, x.device.index)
    scratch = _SKINNY_SCRATCH.get(key)
    if scratch is None or scratch.numel() < need:
        # zero once: every call leaves its tickets zero.  (Allocated outside any graph capture by the warm-up steps a
        # capture is preceded by; a capture that allocates here records the zero fill, which is harmless.)
        scratch = torch.zeros((max(need, 1 << 20),), dtype=torch.float32, device=x.device)
        _SKINNY_SCRATCH[key] = scratch
    with torch.cuda.device(x.device):
        rc = lib.mmfs_linear_skinny(x.data_ptr(), weight.data_ptr(), out.data_ptr(),
                                    residual.data_ptr() if residual is not None else None,
                                    norm_weight.data_ptr() if norm_weight is not None else None, scratch.data_ptr(),
                                    M, N, K, prologue, float(eps), _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "linear_skinny")
    launch_counter[0] += 1
    return out


def conv2d_supported(x: torch.Tensor, weight: torch.Tensor, stride: int, padding: int) -> bool:
    """Whether ``conv2d`` can take this layer (else the caller keeps it on cuDNN: conv_in / conv_out of the UNet)."""
    if x.dtype not in (torch.bfloat16, torch.float16) or not x.is_cuda or x.dim() != 4:
        return False
    B, Cin, H, W = x.shape
    Cout, _, KH, KW = weight.shape
    Ho, Wo = (H + 2 * padding - KH) // stride + 1, (W + 2 * padding - KW) // stride + 1
    tile = (Wo % 16 == 0 and Ho % 8 == 0) or (Wo == 8 and Ho == 8 and B % 2 == 0)
    return Cin % 64 == 0 and Cout % 160 == 0 and stride in (1, 2) and tile


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
    y = torch.empty_like(x, memory_format=torch.channels_last)
    stats = torch.empty((B, 64, groups, 2), dtype=torch.float32, device=x.device)   # per-chunk partial sums
    with torch.cuda.device(x.device):
        rc = _lib.lib().mmfs_groupnorm_nhwc(x.data_ptr(), weight.data_ptr() if weight is not None else None,
                                            bias.data_ptr() if bias is not None else None, y.data_ptr(), stats.data_ptr(),
                                            B, H * W, C, groups, float(eps), int(silu), _DTYPE_CODE[x.dtype], _stream())
    _lib.check(rc, "group_norm_nhwc")
    launch_counter[0] += 2
    return y
