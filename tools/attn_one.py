"""Run the wgmma attention kernel on one BASELINE shape (ncu target) and print CUDA-event timings."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import ops  # noqa: E402

SHAPES = {  # B, H, T, hd, causal
    "llama_cfg3": (4, 40, 2048, 128, True),
    "llama_cfg2": (1, 40, 512, 128, True),
    "clip": (16, 16, 257, 64, False),
    "sd_4096": (2, 5, 4096, 64, False),
    "sd_b16": (16, 5, 4096, 64, False),
    "llama_nc": (4, 40, 2048, 128, False),
}
name = sys.argv[1] if len(sys.argv) > 1 else "llama_cfg3"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
B, H, T, hd, causal = SHAPES[name]
g = torch.Generator(device="cuda").manual_seed(0)
qkv = torch.randn((B, T, 3, H, hd), device="cuda", dtype=torch.bfloat16, generator=g)
q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
for _ in range(2):
    ops.attention(q, k, v, causal=causal)
torch.cuda.synchronize()
ts = []
for _ in range(reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); out = ops.attention(q, k, v, causal=causal); e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
flops = 4.0 * B * H * T * T * hd * (0.5 if causal else 1.0)
t = sorted(ts)[len(ts) // 2] * 1e-3
print(f"{name}: {t * 1e6:.1f} us  {flops / t / 1e12:.1f} TFLOP/s  out mean {out.float().abs().mean().item():.4f}")
