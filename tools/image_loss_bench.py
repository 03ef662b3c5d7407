"""The cost of the image loss's backward through the frozen SD-2.1 UNet.  The full UNet, the full MMFSNet (one
conditioning image's four 1024-channel maps at 64 / 32 / 16 / 8) and the image decoder's Q-Former (77 queries, hidden
1024, over a 512-token 5120-wide context) in bf16 with random weights, at B_I = 4, 8 and 16 images of 512^2 (64^2
latents): the Q-Former, one UNet call with the hook and the MSE against a target -- the part of ``ImageDecoder.forward``
after the VAE encode, which runs under no_grad and is timed by tools/vae_bench.py.  Reports forward-only and
forward+backward medians (CUDA events, after warm-up) and the peak memory; then, from one ``torch.profiler`` run at the
largest batch, the backward's CUDA time per kernel family; then GroupNorm backward alone (achieved bytes/s against the
H100 SXM data sheet's 3.35 TB/s) and the convolution data gradient alone (TFLOP/s).  Prints one JSON line with the card's
name, power limit and SM clocks read in the same run.

    python tools/image_loss_bench.py [--steps N] [--warmup W] [--batches 4,8,16]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import autograd_ops, ops, unet_sd  # noqa: E402
from mm_interleaved_b200.sd_mmfs import MMFSNet  # noqa: E402
from mm_interleaved_b200.visual_tokenizer import PerceiverResampler  # noqa: E402
from tools.attn_bwd_bench import _time, card  # noqa: E402

HBM_PEAK = 3.35e12
BF16 = torch.bfloat16

FAMILIES = [("groupnorm backward", ("gn_bwd",)), ("geglu backward", ("geglu_bwd",)),
            ("conv (wgmma: forward, dgrad)", ("conv_igemm",)), ("attention backward", ("attn_bwd", "dkdv", "dq_kernel")),
            ("msda backward", ("msda_bwd", "ms_deform", "col2im")), ("cudnn", ("cudnn", "conv2d", "implicit_convolve",
                                                                            "xmma", "dgrad", "wgrad")),
            ("cublas", ("nvjet", "gemm", "cutlass", "cublas", "sm90_xmma")), ("layernorm", ("layernorm",))]


def family(name):
    low = name.lower()
    for fam, keys in FAMILIES:
        if any(k in low for k in keys):
            return fam
    return "other"


def build():
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel().to("cuda", BF16).requires_grad_(False)
    net = MMFSNet(1024, tuple(unet.block_out_channels), 2).to("cuda", BF16)
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.02)                   # zero-initialised: would leave the hook without gradient
    qformer = PerceiverResampler(num_queries=77, hidden_size=1024, encoder_hidden_size=5120, num_hidden_layers=1,
                                 num_attention_heads=16, intermediate_size=4096, cross_attention_frequency=1).to("cuda", BF16)
    return unet, net, qformer


def inputs(B, g):
    ctx = torch.randn((B, 512, 5120), device="cuda", generator=g).to(BF16).requires_grad_(True)
    mask = torch.ones((B, 512), device="cuda", dtype=torch.long)
    feats = [torch.randn((B, 1, 1024, s, s), device="cuda", generator=g).to(BF16).requires_grad_(True)
             for s in (64, 32, 16, 8)]
    noisy = torch.randn((B, 4, 64, 64), device="cuda", generator=g).to(BF16).contiguous(memory_format=torch.channels_last)
    target = torch.randn((B, 4, 64, 64), device="cuda", generator=g)
    t = torch.randint(0, 1000, (B,), device="cuda", generator=g)
    return ctx, mask, feats, noisy, target, t


def loss_fn(unet, net, qformer, ctx, mask, feats, noisy, target, t):
    text = qformer(encoder_hidden_states=ctx, encoder_attention_mask=mask)[0]
    pred = unet(noisy, t, text, mmfs_features=feats, mmfs_mask=torch.ones((ctx.shape[0], 1), device="cuda"),
                mmfs_module=net)
    return F.mse_loss(pred.float(), target)


def kernels(iters):
    res = {}
    g = torch.Generator(device="cuda").manual_seed(3)
    for B, C, hw in ((16, 320, 64), (16, 1280, 16)):
        x = torch.randn((B, C, hw, hw), device="cuda", generator=g).to(BF16).contiguous(memory_format=torch.channels_last)
        dy = torch.randn_like(x)
        w, b = torch.ones(C, device="cuda", dtype=BF16), torch.zeros(C, device="cuda", dtype=BF16)
        with torch.no_grad():
            t = _time(lambda: ops.group_norm_nhwc_backward(x, dy, 32, w, b, 1e-5, silu=True), iters)
        nbytes = 6 * x.numel() * 2                                       # x read 3x, dy 2x, dx written once
        res[f"groupnorm_backward_silu_{B}x{C}x{hw}^2"] = {
            "us": round(t * 1e3, 1), "TB_s": round(nbytes / (t * 1e-3) / 1e12, 2),
            "share_of_3.35TB_s": round(nbytes / (t * 1e-3) / HBM_PEAK, 3)}
    for B, cin, cout, hw, stride in ((16, 320, 320, 64, 1), (16, 640, 320, 64, 1), (16, 1280, 1280, 16, 1),
                                     (16, 320, 320, 64, 2)):
        conv = unet_sd.Conv2d(cin, cout, 3, stride=stride, padding=1).to("cuda", BF16).requires_grad_(False)
        ho = hw // stride
        dy = torch.randn((B, cout, ho, ho), device="cuda", generator=g).to(BF16).contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            t = _time(lambda: autograd_ops.conv_input_grad(conv, dy, (B, cin, hw, hw)), iters)
        flops = 2 * B * ho * ho * cout * cin * 9                        # the forward's MACs, what the dgrad redoes
        res[f"conv_dgrad_3x3_s{stride}_{B}x{cin}<-{cout}x{ho}^2"] = {"us": round(t * 1e3, 1),
                                                                       "TFLOP_s": round(flops / (t * 1e-3) / 1e12, 1)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batches", default="4,8,16")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_loss_bench: needs a CUDA device")
    torch.backends.cudnn.deterministic = True
    unet, net, qformer = build()
    res = {"card": card(), "workload": "image loss after the VAE encode: Q-Former (77 queries over 512 x 5120) + SD-2.1 "
           "UNet (frozen) with MMFSNet (4 maps x 1024 ch), bf16, 64^2 latents, MSE"}
    batches = [int(b) for b in a.batches.split(",")]
    for B in batches:
        g = torch.Generator(device="cuda").manual_seed(B)
        args = inputs(B, g)
        params = list(net.parameters()) + list(qformer.parameters())

        def fwd():
            with torch.no_grad():
                loss_fn(unet, net, qformer, *args)

        def fwd_bwd():
            loss_fn(unet, net, qformer, *args).backward()
            for p in params + [args[0], *args[2]]:
                p.grad = None

        out = {}
        for key, fn in (("forward", fwd), ("forward_backward", fwd_bwd)):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            for _ in range(a.warmup):
                fn()
            ts = []
            for _ in range(a.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ts.sort()
            out[key] = {"ms_median": round(ts[len(ts) // 2], 1), "ms_min": round(ts[0], 1), "ms_max": round(ts[-1], 1),
                        "peak_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
        res[f"{B}_images"] = out
    B = batches[-1]
    args = inputs(B, torch.Generator(device="cuda").manual_seed(B))
    loss = loss_fn(unet, net, qformer, *args)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        loss.backward()
        torch.cuda.synchronize()
    per = defaultdict(float)
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[family(ev.key)] += ev.device_time_total / 1e3
    res[f"backward_ms_by_family_{B}_images"] = {k: round(v, 2) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}
    res["kernels"] = kernels(50)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
