"""Dispatch to the wgmma flash-attention kernel (csrc/attn_fwd_sm100.cu)."""
from __future__ import annotations

import os

import torch

from . import _lib
from .msda import _DTYPE_CODE

MIN_QUERY_ROWS = int(os.environ.get("MMFS_ATTN_TC_MIN_ROWS", "16"))   # below this the GEMV-style kernel wins
PERSISTENT = os.environ.get("MMFS_ATTN_PERSISTENT", "1") != "0"         # work-list kernel when items > resident CTAs
_SMS = {}


def supported(q, k, v, Tq, Tkv, hd) -> bool:
    if q.dtype not in (torch.bfloat16, torch.float16) or hd not in (64, 128) or Tq < MIN_QUERY_ROWS:
        return False
    for t in (q, k, v):
        if t.data_ptr() % 16 or t.stride(0) % 8 or t.stride(1) % 8:
            return False
    return q.shape[0] <= 65535 and q.shape[2] <= 65535


def forward(q, k, v, out, key_mask, causal, past, scale):
    B, Tq, H, hd = q.shape
    sms = _SMS.get(q.device.index)
    if sms is None:
        sms = _SMS[q.device.index] = torch.cuda.get_device_properties(q.device).multi_processor_count
    # resident CTAs per SM: 1 at hd 128, 2 at hd 64 (attn_ctas_per_sm in csrc/attn_fwd_sm100.cu); the persistent
    # kernel only pays off with more items than resident CTAs
    if PERSISTENT and B * H * ((Tq + 127) // 128) > (2 if hd == 64 else 1) * sms:
        # one zeroed word per call (a fill kernel; inside a CUDA graph it is re-zeroed on every replay): the kernel's
        # work counter must be private to the launch
        counter = torch.zeros((1,), dtype=torch.int32, device=q.device)
        with torch.cuda.device(q.device):
            rc = _lib.lib().mmfs_attn_forward_persistent(
                q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), key_mask.data_ptr() if key_mask is not None else None,
                B, H, Tq, k.shape[1], hd, q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1),
                out.stride(0), out.stride(1), float(scale), 1 if causal else 0, int(past), _DTYPE_CODE[q.dtype],
                counter.data_ptr(), torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "attention (wgmma, persistent)")
        return
    with torch.cuda.device(q.device):
        rc = _lib.lib().mmfs_attn_forward(
            q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), key_mask.data_ptr() if key_mask is not None else None,
            B, H, Tq, k.shape[1], hd, q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1),
            out.stride(0), out.stride(1), float(scale), 1 if causal else 0, int(past), _DTYPE_CODE[q.dtype],
            torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "attention (wgmma)")
