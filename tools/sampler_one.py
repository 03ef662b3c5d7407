"""Run the fused MMFS sampler on the cfg-3 layer shape (B sequences, masked like the bench step); ncu target."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mm_interleaved_b200 as m  # noqa: E402
from benchmarks.workloads import InterleavedCfg3, msda_algorithmic_bytes  # noqa: E402
from mm_interleaved_b200.mm_interleaved import cross_attention_mask_from_ids  # noqa: E402
from mm_interleaved_b200.mmfs import relative_image_index  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 4
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
masked = (sys.argv[3] if len(sys.argv) > 3 else "masked") == "masked"
mode = sys.argv[4] if len(sys.argv) > 4 else "v2"          # v2 (default kernel) | exact | generic
wl = InterleavedCfg3(0, 1, B)
wl.make_host_inputs(pin=False)
ids = wl.host[0].cuda()
M, D, P, n_lvl, n_img, Lq = 16, 64, 8, 3, 4, 2048
C = M * P * 2 + M * n_lvl * (P + 1)
g = torch.Generator(device="cuda").manual_seed(0)
value = torch.rand((B, n_img * 1344, M, D), device="cuda", generator=g).to(torch.bfloat16)
qproj = torch.randn((B, Lq, C), device="cuda", generator=g)
qproj[..., : M * P * 2] = (torch.rand((B, Lq, M * P * 2), device="cuda", generator=g) * 6 - 3)   # offsets ~ U(-3,3) px
qproj = qproj.to(torch.bfloat16)
rtable = (0.05 * torch.randn((50, C), device="cuda", generator=g)).to(torch.bfloat16)
cross = cross_attention_mask_from_ids(ids, n_img, 1, wl.SOI_ID) if masked else torch.ones((B, Lq, n_img), device="cuda")
relpos = relative_image_index(cross, Lq)
shapes = torch.tensor([(32, 32), (16, 16), (8, 8)] * n_img, device="cuda")
starts = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
ref = torch.full((1, Lq, 1, 2), 0.5, device="cuda")
scale = torch.tensor([2.0, 1.0, 0.5], device="cuda")
flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device="cuda")
kw = dict(v2={}, exact=dict(exact_weights=True), generic=dict(generic=True))[mode]
fn = lambda: m.mmfs_sampler_forward(value, shapes, starts, qproj, rtable, relpos, ref, scale, n_lvl, P, **kw)
for _ in range(3):
    fn()
ts = []
for _ in range(reps):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); out = fn(); e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
t = sorted(ts)[len(ts) // 2] * 1e-3
ab = msda_algorithmic_bytes(B, n_img * 1344, M, D, 12, Lq, P, 2)
print(f"fused sampler B={B} masked={masked} mode={mode}: {t * 1e6:.1f} us  {ab / t / 1e9:.0f} GB/s (sec. 8d bytes)  visible frac {cross.mean().item():.2f}  out {out.float().abs().mean().item():.4f}")
