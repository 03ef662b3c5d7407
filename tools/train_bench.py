"""One training step of the text loss through the 13B Llama-MMFS decoder (40 layers, MMFS cross-attention every 4th,
random weights, bf16) at the cfg-3 sequence (B = 1, T = 2048, 4 images of 1344 feature positions), with the
reference's freezing (only the ``llama_cross_attn`` blocks trainable): ms per forward + backward and peak memory, with
gradient checkpointing off and on, then the per-layer attention kernels (tools/attn_bwd_bench.py).  Prints one JSON
line with the card's name, power limit and SM clocks read in the same run.

    python tools/train_bench.py [--steps N] [--warmup W]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, LlamaModel  # noqa: E402
from tools import attn_bwd_bench  # noqa: E402


def step_ms(model, inputs, steps, warmup):
    def step():
        out = model(**inputs).last_hidden_state
        out.float().pow(2).mean().backward()
        model.zero_grad(set_to_none=True)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated() / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_bench: needs a CUDA device")
    torch.manual_seed(0)
    torch.set_default_dtype(torch.bfloat16)
    with torch.device("cuda"):
        model = LlamaModel(LlamaMMFSConfig())
    torch.set_default_dtype(torch.float32)
    for name, p in model.named_parameters():
        p.requires_grad_("llama_cross_attn" in name)
    B, T, n_img, hw = 1, 2048, 4, 32 * 32 + 16 * 16 + 8 * 8
    g = torch.Generator(device="cuda").manual_seed(1)
    cross = torch.zeros((B, T, n_img), device="cuda")
    for i in range(n_img):                       # image i visible from its position on
        cross[:, i * T // n_img:, i] = 1
    inputs = dict(inputs_embeds=torch.randn((B, T, 5120), device="cuda", generator=g).to(torch.bfloat16),
                  vision_hidden_states=torch.randn((B, n_img, hw, 1024), device="cuda", generator=g).to(torch.bfloat16),
                  attention_mask=torch.ones((B, T), dtype=torch.long, device="cuda"), cross_attention_mask=cross,
                  use_cache=False)
    res = {"card": attn_bwd_bench.card(), "workload": "13B Llama-MMFS decoder, bf16, B=1, T=2048, 4 images, "
           "only llama_cross_attn trainable, loss = mean(h^2)"}
    for ckpt in (False, True):
        model.gradient_checkpointing = ckpt
        ms, gib = step_ms(model, inputs, a.steps, a.warmup)
        res[f"checkpointing_{'on' if ckpt else 'off'}"] = {"ms_per_step": round(ms, 1), "peak_gib": round(gib, 2)}
    res["attention_per_layer"] = attn_bwd_bench.measure(50)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
