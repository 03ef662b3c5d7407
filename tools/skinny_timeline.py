"""Per-CTA timeline of one linear_skinny call (tensor-map kernel, timing probe): kernel entry -> first stage landed ->
last stage landed -> exit, in microseconds relative to the earliest entry."""
import ctypes
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import _lib, ops  # noqa: E402

N, K = int(sys.argv[1]) if len(sys.argv) > 1 else 5120, int(sys.argv[2]) if len(sys.argv) > 2 else 5120
lib = _lib.lib()
assert lib.mmfs_linear_skinny_set_tuning(2 + 4) == 0
g = torch.Generator(device="cuda").manual_seed(0)
x = torch.randn((4, K), device="cuda", dtype=torch.bfloat16, generator=g)
ws = [torch.randn((N, K), device="cuda", dtype=torch.bfloat16, generator=g) for _ in range(4)]
with torch.no_grad():
    for i in range(8):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); ops.linear_skinny(x, ws[i % 4]); e1.record()
        torch.cuda.synchronize()
n_cta = torch.cuda.get_device_properties(0).multi_processor_count   # the kernel runs one CTA per SM
buf = (ctypes.c_ulonglong * (4 * n_cta))()
assert lib.mmfs_linear_skinny_probe(buf, n_cta) == 0
t = torch.tensor(list(buf), dtype=torch.float64).view(n_cta, 4)
t0 = t[:, 0].min()
t = (t - t0) / 1e3
print(f"N={N} K={K} ({N * K * 2 / 1e6:.0f} MB), event time of the last call {e0.elapsed_time(e1) * 1e3:.1f} us")
for name, col in (("entry", 0), ("first stage landed", 1), ("last stage landed", 2), ("exit", 3)):
    c = t[:, col]
    print(f"{name:20s}: min {c.min():6.2f}  median {c.median():6.2f}  max {c.max():6.2f} us")
