"""Fused MMFS sampler on the cfg-3 layer shape (B = 4 sequences, 2048 tokens, 4 images): generic kernel vs the
specialised kernel (fp32 / 16-bit tap weights) over rows-per-warp settings; CUDA events, L2 flushed between runs,
median of `reps`.  Prints one line per setting and a final JSON list."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mm_interleaved_b200 as m  # noqa: E402
from benchmarks.workloads import InterleavedCfg3, msda_algorithmic_bytes  # noqa: E402
from mm_interleaved_b200.mm_interleaved import cross_attention_mask_from_ids  # noqa: E402
from mm_interleaved_b200.mmfs import _relative_image_index  # noqa: E402
from mm_interleaved_b200.sampler import set_sampler_tuning  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
B = 4
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
shapes = torch.tensor([(32, 32), (16, 16), (8, 8)] * n_img, device="cuda")
starts = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
ref = torch.full((1, Lq, 1, 2), 0.5, device="cuda")
scale = torch.tensor([2.0, 1.0, 0.5], device="cuda")
flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device="cuda")
ab = msda_algorithmic_bytes(B, n_img * 1344, M, D, 12, Lq, P, 2)
rows = []
for masked in (True, False):
    cross = cross_attention_mask_from_ids(ids, n_img, 1, wl.SOI_ID) if masked else torch.ones((B, Lq, n_img), device="cuda")
    relpos = _relative_image_index(cross, Lq)
    for mode, rpws in (("generic", (0,)), ("generic_w16", (0,)), ("exact", (0,)), ("exact_occ4", (0,)), ("v2", (0, 1, 2, 4, 8)),
                       ("v2_occ4", (0, 1, 2, 4, 8))):
        kw = dict(v2={}, v2_occ4={}, exact=dict(exact_weights=True), exact_occ4=dict(exact_weights=True), generic=dict(generic=True),
                  generic_w16=dict(generic=True, w16=True))[mode]
        for rpw in rpws:
            set_sampler_tuning(rpw, 1, 4 if mode.endswith("occ4") else 3)
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
            row = dict(masked=masked, visible_frac=round(float(cross.mean()), 3), mode=mode, rows_per_warp=rpw,
                       us=round(t * 1e6, 1), gbs_8d=round(ab / t / 1e9, 1), frac_hbm=round(ab / t / 1e9 / 6584.5, 4))
            rows.append(row)
            print(row, flush=True)
set_sampler_tuning(0, 1, 3)
print(json.dumps(rows))
