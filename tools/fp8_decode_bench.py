"""FP8 decoding against bf16 on the Llama-13B MMFS decoder (random weights), in one run:

  kernels: each decode linear (fused QKV, o_proj, fused gate/up, down_proj, the folded head) at M in {1, 5, 20} rows,
           ``ops.linear_fp8`` against the bf16 cuBLAS GEMM (``torch.matmul`` into the same output; CUDA events over 200 launches after 20 warm-up ones;
           bytes/s from the shapes: weights + x + output);
  decode:  graphed ms per token of greedy and 5-beam decoding at the caption prompt (1 image in 80 tokens) and the
           2048-token 4-image prompt of tools/beam_bench.py, B = 1, bf16 against ``enable_fp8_decode()``, the two
           alternating.  ms per token = (time of a 20-token call - time of a 1-token call) / 19, each the best of 2.

Prints one JSON object with the card name, its power limit and SM clock read in the same run.

    python tools/fp8_decode_bench.py
"""
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchmarks import workloads  # noqa: E402
from mm_interleaved_b200 import ops  # noqa: E402
from mm_interleaved_b200.mm_interleaved import InterleavedForward  # noqa: E402

SHAPES = {"qkv": (15360, 5120), "o_proj": (5120, 5120), "gate_up": (27648, 5120), "down_proj": (5120, 13824),
          "head": (32128, 5120)}
MAX_NEW, NB = 20, 5


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        out = []
    row = out[torch.cuda.current_device()] if len(out) > torch.cuda.current_device() else ""
    return {"card": torch.cuda.get_device_name(), "nvidia_smi": dict(zip(q.split(","), [s.strip() for s in row.split(",")]))}


def timed(fn, iters):
    for _ in range(20):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / iters


def caption_inputs(B):
    """tools/beam_bench.py's caption prompt: 1 image (64 image tokens after <soi>) in an 80-token prompt."""
    g = torch.Generator().manual_seed(77)
    W = workloads.InterleavedCfg3
    ids = torch.randint(3, 31999, (B, 80), generator=g)
    ids[:, 0] = workloads.BOS_ID
    ids[:, 1] = W.SOI_ID
    ids[:, 2:2 + W.TOK_PER_IMG] = W.IMG_ID
    return ids, torch.rand((B, 3, 224, 224), generator=g), torch.ones(B, dtype=torch.long), 1


def long_inputs(B):
    """tools/beam_bench.py's long prompt: 2048 tokens, 4 images."""
    wl = workloads.InterleavedCfg3(0, 1, B)
    wl.make_host_inputs(pin=False)
    ids, img, nimg = wl.host
    return ids, img, nimg, wl.N_IMG


def kernel_rows(rows):
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (N, K) in SHAPES.items():
        w = (torch.randn((N, K), generator=g, device="cuda") * 0.02).to(torch.bfloat16)
        w8, s = ops.quantize_fp8_per_channel(w)
        for M in (1, 5, 20):
            x = torch.randn((M, K), generator=g, device="cuda").to(torch.bfloat16)
            out = torch.empty((M, N), dtype=torch.bfloat16, device="cuda")
            us_fp8 = timed(lambda: ops.linear_fp8(x, w8, s, out=out), 200)
            us_bf16 = timed(lambda: torch.matmul(x, w.t(), out=out), 200)
            act = 2 * M * (K + N)
            rows[f"{name}_M{M}_fp8_us"] = us_fp8
            rows[f"{name}_M{M}_bf16_us"] = us_bf16
            rows[f"{name}_M{M}_fp8_GBps"] = (N * K + act) / us_fp8 / 1e3
            rows[f"{name}_M{M}_bf16_GBps"] = (2 * N * K + act) / us_bf16 / 1e3
            rows[f"{name}_M{M}_speedup"] = us_bf16 / us_fp8
        del w, w8, s
    torch.cuda.empty_cache()


def decode_rows(rows, model):
    eos = [2, workloads.InterleavedCfg3.SOI_ID]
    for shape, make in (("caption", caption_inputs), ("long", long_inputs)):
        ids, img, nimg, n_img = make(1)
        ids, img, nimg = ids.cuda(), img.cuda(), nimg.cuda()
        vis = model._tokenize(img)
        for beams in (1, NB):
            def per_token(fp8):
                gen = lambda n: InterleavedForward.generate_texts(model, ids, vis, nimg, n_img, max_new_tokens=n,
                                                                  eos_token_id=eos, min_length=8, num_beams=beams)
                model.enable_fp8_decode(fp8)
                model.enable_decode_graphs(True)
                best, out = {}, None
                for n in (MAX_NEW, 1):
                    for _ in range(2):
                        torch.cuda.synchronize(); t0 = time.time()
                        o = gen(n)
                        torch.cuda.synchronize(); dt = time.time() - t0
                        best[n] = min(best.get(n, dt), dt)
                        out = o if n == MAX_NEW else out
                model.enable_decode_graphs(False)
                torch.cuda.empty_cache()
                return 1e3 * (best[MAX_NEW] - best[1]) / (MAX_NEW - 1), out

            key = f"{shape}_{'greedy' if beams == 1 else f'beam{beams}'}"
            bf16, fp8 = [], []
            for _ in range(2):                                              # alternating
                t, out_b = per_token(False)
                bf16.append(t)
                t, out_f = per_token(True)
                fp8.append(t)
            rows[f"{key}_prompt_tokens"] = ids.shape[1]
            rows[f"{key}_bf16_ms_per_token"] = min(bf16)
            rows[f"{key}_fp8_ms_per_token"] = min(fp8)
            rows[f"{key}_bf16_runs"], rows[f"{key}_fp8_runs"] = bf16, fp8
            rows[f"{key}_ids_equal"] = bool(torch.equal(out_b, out_f))
        model.enable_fp8_decode(False)
        del vis
        torch.cuda.empty_cache()


rows = card()
with torch.no_grad():
    kernel_rows(rows)
    if "--kernels" not in sys.argv:
        decode_rows(rows, workloads.full_model(with_image_decoder=False))
rows.update(card())
print(json.dumps(rows))
