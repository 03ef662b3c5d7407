"""Micro-benchmark of the MSDA forward kernel over the BASELINE shapes.
CUDA-event timing on the launching stream, L2 flushed between iterations.  Internal tool
(bench.py is the contract); results land in gpurun_out/msda_sweep.json."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mm_interleaved_b200 as m  # noqa: E402
from oracle import make_msda_inputs  # noqa: E402

SHAPES = {
    "cfg3_llm_L12_Lq2048": (1, [(32, 32), (16, 16), (8, 8)] * 4, 16, 64, 2048, 8),
    "cfg3_llm_x4seq": (4, [(32, 32), (16, 16), (8, 8)] * 4, 16, 64, 2048, 8),
    "cfg2_llm_L3_Lq512": (1, [(32, 32), (16, 16), (8, 8)], 16, 64, 512, 8),
    "sd_Lq4096": (1, [(64, 64), (32, 32), (16, 16), (8, 8)], 16, 64, 4096, 8),
    "sd_Lq4096_x16": (16, [(64, 64), (32, 32), (16, 16), (8, 8)], 16, 64, 4096, 8),
    "sd_Lq1024": (1, [(64, 64), (32, 32), (16, 16), (8, 8)], 16, 64, 1024, 8),
    "sd_Lq64": (1, [(64, 64), (32, 32), (16, 16), (8, 8)], 16, 64, 64, 8),
    "adapter_inj": (4, [(32, 32), (16, 16), (8, 8)], 16, 32, 256, 4),
    "decode_Lq1": (8, [(32, 32), (16, 16), (8, 8)] * 4, 16, 64, 1, 8),
}


def algo_bytes(N, shapes, M, D, Lq, P, es):
    S = sum(h * w for h, w in shapes)
    L = len(shapes)
    return es * (N * S * M * D + 3 * N * Lq * M * L * P + N * Lq * M * D) + 24 * L


def time_kernel(fn, iters=20, flush=None):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2] * 1e-3, ts[0] * 1e-3


def main():
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    res = []
    for name, (N, shapes, M, D, Lq, P) in SHAPES.items():
        for loc_mode in ("llm", "clustered"):
            for dtype in (torch.bfloat16, torch.float32):
                v, s, st, loc, a = make_msda_inputs(N, shapes, M, D, Lq, P, seed=0, loc_mode="clustered" if loc_mode == "llm" else loc_mode, dtype=dtype)
                if loc_mode == "llm":
                    # MMFS LLM flavour: reference point (0.5, 0.5) + offsets ~ U(-3,3)/16 (bias init) + noise,
                    # identical across the 3 levels of an image
                    g = torch.Generator().manual_seed(1)
                    nimg = max(len(shapes) // 3, 1)
                    off = (torch.rand((N, Lq, M, nimg, 1, P, 2), generator=g) * 6 - 3) / 16.0
                    off = off + 0.03 * torch.randn((N, Lq, M, nimg, 1, P, 2), generator=g)
                    loc = (0.5 + off).expand(N, Lq, M, nimg, len(shapes) // nimg, P, 2).reshape(N, Lq, M, len(shapes), P, 2)
                if name.startswith("sd"):
                    # SD flavour: pixel-grid reference points + small offsets
                    side = int(Lq ** 0.5)
                    ys, xs = torch.meshgrid(torch.arange(side), torch.arange(side), indexing="ij")
                    ref = torch.stack([(xs.flatten() + 0.5) / side, (ys.flatten() + 0.5) / side], -1)
                    loc = ref[None, :, None, None, None, :] + (loc - 0.5) * (12.0 / side if loc_mode == "clustered" else 0.5)
                args = [v.to("cuda", dtype), s.cuda(), st.cuda(), loc.to("cuda", dtype).contiguous(), a.to("cuda", dtype)]
                ab = algo_bytes(N, shapes, M, D, Lq, P, 2 if dtype == torch.bfloat16 else 4)
                fn = lambda: m.ms_deform_attn_forward(*args, 64)
                med_cold, best_cold = time_kernel(fn, flush=flush)
                med_warm, best_warm = time_kernel(fn, flush=None)
                r = dict(shape=name, loc=loc_mode, dtype=str(dtype).split(".")[-1],
                         algo_MB=ab / 1e6, cold_us=med_cold * 1e6, warm_us=med_warm * 1e6,
                         cold_GBs=ab / med_cold / 1e9, warm_GBs=ab / med_warm / 1e9)
                res.append(r)
                print(json.dumps(r), flush=True)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "gpurun_out", "msda_sweep.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
