"""Dispatch to the wgmma flash-attention kernel (csrc/attn_fwd_sm100.cu)."""
from __future__ import annotations

import torch

from . import _lib
from .msda import _DTYPE_CODE

MIN_QUERY_ROWS = 16   # below this the GEMV-style kernel wins


def supported(q, k, v, Tq, Tkv, hd) -> bool:
    if q.dtype not in (torch.bfloat16, torch.float16) or hd not in (64, 128) or Tq < MIN_QUERY_ROWS:
        return False
    for t in (q, k, v):
        if t.data_ptr() % 16 or t.stride(0) % 8 or t.stride(1) % 8:
            return False
    return q.shape[0] <= 65535 and q.shape[2] <= 65535


def forward(q, k, v, out, key_mask, causal, past, scale):
    B, Tq, H, hd = q.shape
    # scratch for the persistent kernel's work counter: the library zeroes it itself when it runs persistent
    counter = torch.empty((1,), dtype=torch.int32, device=q.device)
    with torch.cuda.device(q.device):
        rc = _lib.lib().mmfs_attn_forward(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), key_mask.data_ptr() if key_mask is not None else None,
            B, H, Tq, k.shape[1], hd, q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1),
            out.stride(0), out.stride(1), float(scale), 1 if causal else 0, int(past), _DTYPE_CODE[q.dtype],
            counter.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "attention (wgmma)")
