"""The cost of training the ViT-Adapter with the visual tokenizer's head.  The full-size tokenizer (CLIP ViT-L/14 +
ViT-Adapter + 12-layer qk-norm Q-Former, bf16, random weights) on 4 and on 16 images at 224^2: forward and backward of a
seeded projection of all its outputs, timed with CUDA events with (a) adapter and head trainable
(``freeze_like_reference``) and (b) the head only, alternating, with the peak memory of each.  Then the two new kernels
alone over many launches at the 16-image shapes: time and achieved HBM bytes/s (bytes computed from the shapes below)
against the H100 SXM data sheet's 3.35 TB/s.  Prints one JSON line with the card's name, power limit and SM clocks read
in the same run.

    python tools/adapter_bwd_bench.py [--steps N] [--warmup W]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import ops  # noqa: E402
from mm_interleaved_b200.visual_tokenizer import VisualTokenizer  # noqa: E402
from tools.attn_bwd_bench import _time, card  # noqa: E402

HBM_PEAK = 3.35e12


def kernels(iters):
    """quick-GELU backward over one CLIP MLP activation (16 x 257 tokens x 4096) and the three output-resize backwards
    (16 images x 1024 channels, 16^2 stage maps, dy in the token layout), bf16."""
    g = torch.Generator(device="cuda").manual_seed(2)
    res = {}
    h = torch.randn((16 * 257, 4096), device="cuda", generator=g).to(torch.bfloat16)
    dy = torch.randn_like(h)
    with torch.no_grad():
        t = _time(lambda: ops.quick_gelu_backward(h, dy), iters)
    nbytes = 3 * h.numel() * 2                                           # read h and dy, write dh
    res["quick_gelu_backward_16x257x4096"] = {"us": round(t * 1e3, 1), "TB_s": round(nbytes / (t * 1e-3) / 1e12, 2),
                                              "share_of_3.35TB_s": round(nbytes / (t * 1e-3) / HBM_PEAK, 3)}
    B, C, side = 16, 1024, 16
    for f in (4, 2, 0.5):
        o = int(side * f)
        d = torch.randn((B, o * o, C), device="cuda", generator=g).to(torch.bfloat16).transpose(1, 2).reshape(B, C, o, o)
        with torch.no_grad():
            t = _time(lambda: ops.resize_bilinear_backward(d, (side, side), f), iters)
        nbytes = (B * C * o * o + B * C * side * side) * 2                # read dy once, write dx once
        res[f"resize_backward_x{f}_16x1024x{side}^2"] = {
            "us": round(t * 1e3, 1), "TB_s": round(nbytes / (t * 1e-3) / 1e12, 2),
            "share_of_3.35TB_s": round(nbytes / (t * 1e-3) / HBM_PEAK, 3)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adapter_bwd_bench: needs a CUDA device")
    torch.manual_seed(0)
    torch.backends.cudnn.deterministic = True
    tok = VisualTokenizer().to("cuda", torch.bfloat16).freeze_like_reference()
    adapter = [p for n, p in tok.named_parameters() if n.startswith("encoder.") and p.requires_grad]
    with torch.no_grad():
        for blk in tok.encoder.vision_model.adapter_interactions:
            blk.injector.gamma.fill_(0.5)                  # zero-initialised: would leave the injectors without gradient
    res = {"card": card(), "workload": "VisualTokenizer (ViT-L/14 + adapter + 12-layer Q-Former), bf16, 224^2, loss = "
           "seeded projection of vis_embed, image_embeds and the 4 multi-scale maps"}
    for n_img in (4, 16):
        g = torch.Generator(device="cuda").manual_seed(n_img)
        images = torch.rand((n_img, 3, 224, 224), device="cuda", generator=g).to(torch.bfloat16)
        with torch.no_grad():
            shapes = [o.shape for o in (lambda r: [r["vis_embed"], r["image_embeds"], *r["multiscale_features"]])(tok(images))]
        proj = [torch.randn(s, device="cuda", generator=g).to(torch.bfloat16) for s in shapes]

        def step():
            r = tok(images)
            outs = [r["vis_embed"], r["image_embeds"], *r["multiscale_features"]]
            sum((o.float() * p.float()).sum() for o, p in zip(outs, proj)).backward()
            tok.zero_grad(set_to_none=True)

        times = {"adapter_and_head": [], "head_only": []}
        peak = {}
        for key in times:                                   # warm-up of both variants, with the peak memory of each
            for p in adapter:
                p.requires_grad_(key == "adapter_and_head")
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            for _ in range(a.warmup):
                step()
            torch.cuda.synchronize()
            peak[key] = torch.cuda.max_memory_allocated()
        for _ in range(a.steps):                            # alternate, one step each
            for key in times:
                for p in adapter:
                    p.requires_grad_(key == "adapter_and_head")
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step()
                e1.record()
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1))
        for key, ts in times.items():
            ts = sorted(ts)
            res[f"{n_img}_images_{key}"] = {"ms_median": round(ts[len(ts) // 2], 1), "ms_min": round(ts[0], 1),
                                            "ms_max": round(ts[-1], 1), "peak_GiB": round(peak[key] / 2 ** 30, 2)}
        for p in adapter:
            p.requires_grad_(True)
    res["kernels"] = kernels(200)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
