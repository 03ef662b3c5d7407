"""Time the reference's own CUDA op (oracle/_ref, compiled unmodified for sm_90a) against this repo's kernel on the
same H100, same inputs (fp16 and fp32 -- the reference has no bf16 dispatch).  CUDA events, L2 flushed."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mm_interleaved_b200 as m  # noqa: E402
from oracle import make_msda_inputs, ref_cuda  # noqa: E402
from tools.msda_sweep import SHAPES, algo_bytes, time_kernel  # noqa: E402

ref = ref_cuda.load()
flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device="cuda")
rows = []
for name in ("cfg3_llm_L12_Lq2048", "cfg3_llm_x4seq", "cfg2_llm_L3_Lq512", "sd_Lq4096", "sd_Lq4096_x16", "sd_Lq1024", "sd_Lq64", "adapter_inj", "decode_Lq1"):
    N, shapes, M, D, Lq, P = SHAPES[name]
    for dtype in (torch.float16, torch.float32):
        v, s, st, loc, a = make_msda_inputs(N, shapes, M, D, Lq, P, seed=0, loc_mode="clustered", dtype=dtype)
        args = [v.to("cuda", dtype), s.cuda(), st.cuda(), loc.to("cuda", dtype), a.to("cuda", dtype)]
        t_ref, _ = time_kernel(lambda: ref.ms_deform_attn_forward(*args, 1), iters=10, flush=flush)     # im2col_step = 1 as every caller sets it
        t_our, _ = time_kernel(lambda: m.ms_deform_attn_forward(*args, 1), iters=10, flush=flush)
        d = (ref.ms_deform_attn_forward(*args, 1).float() - m.ms_deform_attn_forward(*args, 1).float()).abs().max().item()
        ab = algo_bytes(N, shapes, M, D, Lq, P, 2 if dtype == torch.float16 else 4)
        r = dict(shape=name, dtype=str(dtype).split(".")[-1], ref_us=t_ref * 1e6, ours_us=t_our * 1e6, speedup=t_ref / t_our,
                 ours_GBs=ab / t_our / 1e9, ref_GBs=ab / t_ref / 1e9, max_abs_diff=d)
        rows.append(r)
        print(json.dumps(r), flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(rows, open(os.path.join(ROOT, "gpurun_out", "ref_vs_ours.json"), "w"), indent=1)
