"""A/B for the Llama dense linears: this repo's wgmma implicit-GEMM mainloop at KH = KW = 1 (which IS a plain GEMM:
M = 128-pixel tiles, N = 160, K = 64 per stage, one CTA per SM) against cuBLAS (torch F.linear) on the decoder's shapes,
same GPU, CUDA events, median of `reps`.  Prints one JSON object."""
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import ops  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
dt = torch.bfloat16
rows = []
flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def timeit(fn):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2] * 1e-3


M = 8192                                            # 4 sequences x 2048 tokens
for name, N, K in (("qkv_proj", 15360, 5120), ("o_proj", 5120, 5120), ("down_proj", 5120, 13824), ("gate_up (N padded to 27680)", 27680, 5120)):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn((M, K), device="cuda", generator=g) * 0.5).to(dt)
    w = (torch.randn((N, K), device="cuda", generator=g) * 0.02).to(dt)
    t_lib = timeit(lambda: F.linear(x, w))
    # the same GEMM through the convolution kernel: M = 64 "images" of 8 x 16 pixels, 1x1 filter
    xi = x.view(64, 8, 16, K).permute(0, 3, 1, 2)   # NCHW view of NHWC storage = channels_last
    wk = w.view(N, 1, 1, K)
    ok = ops.conv2d_supported(xi, w.view(N, K, 1, 1), 1, 0)
    t_own, err = None, None
    if ok:
        t_own = timeit(lambda: ops.conv2d(xi, wk, None, 1, 0))
        ref = F.linear(x, w).float()
        got = ops.conv2d(xi, wk, None, 1, 0).permute(0, 2, 3, 1).reshape(M, N).float()
        err = float((got - ref).abs().max() / ref.abs().max())
    fl = 2.0 * M * N * K
    rows.append(dict(layer=name, M=M, N=N, K=K, cublas_us=round(t_lib * 1e6, 1), cublas_tflops=round(fl / t_lib / 1e12, 1),
                     own_us=None if t_own is None else round(t_own * 1e6, 1),
                     own_tflops=None if t_own is None else round(fl / t_own / 1e12, 1), rel_err=err))
    print(rows[-1], flush=True)
print(json.dumps(rows))
