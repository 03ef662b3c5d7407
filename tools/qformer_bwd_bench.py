"""The cost of training the visual tokenizer's head (pos_proj, pos_ln, post_ln, the 12-layer qk-norm Q-Former, proj) with
the text loss.  One step = the full-size tokenizer (CLIP ViT-L/14 + ViT-Adapter frozen) on 4 images at 224^2, its
vis_embed spliced into the 13B Llama-MMFS decoder's input (B = 1, T = 2048, 64 positions per image), forward and
backward of a mean-square loss with only the ``llama_cross_attn`` blocks trainable (tools/train_bench.py's step),
timed with the head trainable and frozen, alternating.  Then the Q-Former's two attention shapes alone (4 images x 12
heads x hd 64, bf16, non-causal): self-attention Tq = Tkv = 64 and cross-attention Tq = 64, Tkv = 257, forward with LSE
and backward, CUDA events over many launches.  Prints one JSON line with the card's name, power limit and SM clocks
read in the same run.  Random weights, bf16.

    python tools/qformer_bwd_bench.py [--steps N] [--warmup W]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import ops  # noqa: E402
from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, LlamaModel  # noqa: E402
from mm_interleaved_b200.visual_tokenizer import VisualTokenizer  # noqa: E402
from tools.attn_bwd_bench import _time, card  # noqa: E402


def attention_shapes(iters):
    B, H, hd = 4, 12, 64
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {}
    for name, Tkv in (("self_64x64", 64), ("cross_64x257", 257)):
        q = torch.randn((B, 64, H, hd), device="cuda", generator=g).to(torch.bfloat16)
        k, v = (torch.randn((B, Tkv, H, hd), device="cuda", generator=g).to(torch.bfloat16) for _ in range(2))
        d_out = torch.randn_like(q)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        with torch.no_grad():
            out, lse = ops.attention_forward_lse(q, k, v, causal=False)
            fwd = _time(lambda: ops.attention_forward_lse(q, k, v, causal=False), iters)
            bwd = _time(lambda: ops.attention_backward_general(q, k, v, out, d_out, lse, dq, dk, dv), iters)
        res[name] = {"forward_lse_us": round(fwd * 1e3, 1), "backward_us": round(bwd * 1e3, 1)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qformer_bwd_bench: needs a CUDA device")
    torch.manual_seed(0)
    torch.set_default_dtype(torch.bfloat16)
    with torch.device("cuda"):
        model = LlamaModel(LlamaMMFSConfig())
    torch.set_default_dtype(torch.float32)
    tok = VisualTokenizer().to("cuda", torch.bfloat16)
    for name, p in model.named_parameters():
        p.requires_grad_("llama_cross_attn" in name)
    tok.encoder.requires_grad_(False)
    B, T, n_img, hw = 1, 2048, 4, 32 * 32 + 16 * 16 + 8 * 8
    g = torch.Generator(device="cuda").manual_seed(1)
    images = torch.rand((n_img, 3, 224, 224), device="cuda", generator=g).to(torch.bfloat16)
    embeds = torch.randn((B, T, 5120), device="cuda", generator=g).to(torch.bfloat16)
    pos = torch.cat([torch.arange(64, device="cuda") + 16 + i * T // n_img for i in range(n_img)])   # image token slots
    cross = torch.zeros((B, T, n_img), device="cuda")
    for i in range(n_img):
        cross[:, i * T // n_img:, i] = 1
    kw = dict(vision_hidden_states=torch.randn((B, n_img, hw, 1024), device="cuda", generator=g).to(torch.bfloat16),
              attention_mask=torch.ones((B, T), dtype=torch.long, device="cuda"), cross_attention_mask=cross, use_cache=False)

    def step():
        vis = tok(images)["vis_embed"].reshape(1, -1, 5120)
        e = embeds.index_copy(1, pos, vis)
        model(inputs_embeds=e, **kw).last_hidden_state.float().pow(2).mean().backward()
        model.zero_grad(set_to_none=True)
        tok.zero_grad(set_to_none=True)

    head = [p for n, p in tok.named_parameters() if not n.startswith("encoder.") and n != "pos_embed"]
    times = {"head_trainable": [], "head_frozen": []}
    for trainable in (True, False):                      # warm-up of both variants
        for p in head:
            p.requires_grad_(trainable)
        for _ in range(a.warmup):
            step()
    for _ in range(a.steps):                             # alternate, one step each
        for trainable, key in ((True, "head_trainable"), (False, "head_frozen")):
            for p in head:
                p.requires_grad_(trainable)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            torch.cuda.synchronize()
            times[key].append(e0.elapsed_time(e1))
    res = {"card": card(), "workload": "tokenizer (4 x 224^2, encoder frozen) + 13B Llama-MMFS decoder, bf16, B=1, "
           "T=2048, only llama_cross_attn (+ tokenizer head) trainable, loss = mean(h^2)"}
    for key, ts in times.items():
        ts = sorted(ts)
        res[key] = {"ms_median": round(ts[len(ts) // 2], 1), "ms_min": round(ts[0], 1), "ms_max": round(ts[-1], 1)}
    res["qformer_attention_4x12x64"] = attention_shapes(200)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
