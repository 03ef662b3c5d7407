"""Time the training-path attention kernels of one Llama-13B layer at the cfg-3 sequence (B = 1, 40 heads, T = 2048,
hd 128, bf16, causal): mmfs_attn_forward_lse and mmfs_attn_backward, CUDA events over many launches.  Prints one JSON
line with the card's name, power limit and SM clocks read in the same run.

Algorithmic FLOPs: the causal forward does 2 * B * H * T^2 * hd (QK^T and PV over half the score matrix); the backward
counts 2.5x that (dV, dP, dQ, dK plus half a recomputed S), as flash-attention papers do, although this kernel
recomputes P twice.  Share of peak is against the data sheet's 989 dense BF16 TFLOP/s (H100 SXM at 700 W).

    python tools/attn_bwd_bench.py [--iters N]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import ops  # noqa: E402

PEAK_TFLOPS = 989.0


def card():
    """Name, power limit and current / max SM clock of device 0, read now."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit not read"


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def measure(iters):
    """Per-layer timings of the causal attention forward (with LSE) and backward at the 13B cfg-3 shape."""
    B, H, T, hd = 1, 40, 2048, 128
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn((B, T, 3, H, hd), device="cuda", generator=g).to(torch.bfloat16)
    d_out = torch.randn((B, T, H, hd), device="cuda", generator=g).to(torch.bfloat16)
    dqkv = torch.empty_like(qkv)
    q, k, v = qkv.unbind(2)
    with torch.no_grad():
        out, lse = ops.attention_forward_lse(q, k, v)
        fwd_ms = _time(lambda: ops.attention_forward_lse(q, k, v), iters)
        bwd_ms = _time(lambda: ops.attention_backward(q, k, v, out, d_out, lse, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2]),
                       iters)
    fwd_flops = 2.0 * B * H * T * T * hd
    bwd_tflops = 2.5 * fwd_flops / (bwd_ms * 1e-3) / 1e12
    return {
        "shape": {"B": B, "H": H, "T": T, "hd": hd, "dtype": "bf16", "causal": True},
        "forward_lse_ms": round(fwd_ms, 4), "forward_lse_tflops": round(fwd_flops / (fwd_ms * 1e-3) / 1e12, 1),
        "backward_ms": round(bwd_ms, 4), "backward_tflops": round(bwd_tflops, 1),
        "backward_share_of_989": round(bwd_tflops / PEAK_TFLOPS, 3),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_bwd_bench: needs a CUDA device")
    print(json.dumps({"card": card(), **measure(a.iters)}))


if __name__ == "__main__":
    main()
