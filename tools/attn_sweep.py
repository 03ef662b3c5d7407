"""Per-CTA fixed cost vs per-tile cost of the wgmma attention kernel: time non-causal and causal problems of different
lengths with the number of work items held near 2560 and fit  t_cta = c0 + n_tiles * t_tile, where the CTA slots are the
resident CTAs of the hd-128 kernel (one per SM)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import ops  # noqa: E402

g = torch.Generator(device="cuda").manual_seed(0)
hd = 128
slots = torch.cuda.get_device_properties(0).multi_processor_count   # 1 resident CTA per SM at hd 128
rows = []
for causal in (False, True):
    for T in (256, 512, 1024, 2048, 4096):
        q_tiles = T // 128
        BH = max(1, 2560 // q_tiles)
        B, H = (BH // 40, 40) if BH >= 40 else (1, BH)
        qkv = torch.randn((B, T, 3, H, hd), device="cuda", dtype=torch.bfloat16, generator=g)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        for _ in range(3):
            ops.attention(q, k, v, causal=causal)
        torch.cuda.synchronize()
        ts = []
        for _ in range(9):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); ops.attention(q, k, v, causal=causal); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        t = sorted(ts)[len(ts) // 2]
        n_cta = B * H * q_tiles
        tiles = sum(min(2 * (i + 1), T // 64) if causal else T // 64 for i in range(q_tiles)) * B * H
        flops = 4.0 * B * H * T * T * hd * (0.5 if causal else 1.0)
        rows.append((causal, T, n_cta, tiles, t))
        print(f"causal={int(causal)} T={T:5d} B={B:3d} H={H:3d} ctas={n_cta:5d} key-tiles={tiles:7d}: {t:8.1f} us  {flops / t / 1e6:7.1f} TFLOP/s  "
              f"{t * slots / n_cta:6.2f} us per CTA slot-time, {t * slots / tiles:6.3f} us per tile")
