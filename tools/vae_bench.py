"""SD-2.1 VAE decode timing: a bf16 decode of (8, 4, 64, 64) latents (eight 512 x 512 images) at SD-2.1 widths.
With ``--encode``, the encoder half instead (see ``encode_bench``): eight 512 x 512 images encoded in bf16 on this
repo's kernels, on cuDNN (``unet_sd.USE_CONV_KERNEL = False``) and in fp32; the three downsample shapes against
``F.pad`` + cuDNN; cuDNN's ``conv_in`` (Cin = 3) alone; one ``ImageDecoder.forward`` (the image loss) with B_I = 8.

    python tools/vae_bench.py [--encode] [--batch 8] [--iters 10] [--warmup 3] [--out DIR]

* whole decode, CUDA events after warm-up, median (and min / max) of ``--iters`` decodes, for three paths of the same
  module and weights: bf16 on this repo's kernels; bf16 on cuDNN (``unet_sd.USE_CONV_KERNEL = False``: every
  convolution, the upsamplers as interpolate + conv, and GroupNorm on torch); fp32 on cuDNN (the reference's
  precision, PyTorch's default TF32 settings, reported);
* per convolution shape of the decode: kernel time (CUDA events over repeated launches of the one op) and TFLOP/s from
  the shape, own kernel vs cuDNN (channels_last bf16).  The fused upsample convolution is counted at its own 4-tap
  FLOPs; the 9-tap count of interpolate + conv3x3 (the cuDNN path's work) is printed beside it.
Prints the card's name, power limit and max SM clock, and one JSON line; ``--out`` also writes it to DIR/vae_bench.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mm_interleaved_b200 import ops, unet_sd  # noqa: E402
from mm_interleaved_b200.vae_sd import AutoencoderKL, Upsample2D  # noqa: E402

CL = torch.channels_last


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "nvidia-smi unavailable"


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def kernel_ms(fn, reps=20):
    """Mean time of one launch of ``fn`` over ``reps`` back-to-back launches (after one warm-up launch)."""
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def conv_shapes(model, z):
    """(kind, B, Cin, Cout, H, W, k) of every convolution the decode runs, with its input shape: 'conv' or 'up2x'."""
    seen = []
    hooks = []
    for mod in model.modules():
        if isinstance(mod, Upsample2D):
            hooks.append(mod.register_forward_pre_hook(
                lambda mod, args: seen.append(("up2x",) + tuple(args[0].shape[:2]) + (mod.conv.out_channels,) + tuple(args[0].shape[2:]) + (3,))))
    conv_of_up = {id(mod.conv) for mod in model.modules() if isinstance(mod, Upsample2D)}
    for mod in model.modules():
        if isinstance(mod, torch.nn.Conv2d) and id(mod) not in conv_of_up:
            hooks.append(mod.register_forward_pre_hook(
                lambda mod, args: seen.append(("conv",) + tuple(args[0].shape[:2]) + (mod.out_channels,) + tuple(args[0].shape[2:]) + (mod.kernel_size[0],))))
    # the hooks see nn.Conv2d.__call__ only on the cuDNN path; run it once there to list every layer
    unet_sd.USE_CONV_KERNEL = False
    try:
        model.decode(z)
    finally:
        unet_sd.USE_CONV_KERNEL = True
        for h in hooks:
            h.remove()
    counts = {}
    for s in seen:
        counts[s] = counts.get(s, 0) + 1
    return counts


def _median(t):
    return {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t)}


def encode_bench(args, info):
    """``--encode``: the encoder half and the image-decoder loss step it feeds."""
    from mm_interleaved_b200.mm_interleaved import ImageDecoder
    torch.manual_seed(0)
    model = AutoencoderKL(with_encoder=True).eval().to("cuda", torch.bfloat16).to(memory_format=CL)
    x = torch.rand((args.batch, 3, 512, 512), device="cuda") * 2 - 1
    res = {"gpu": info, "mode": "encode", "batch": args.batch, "iters": args.iters,
           "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "matmul_allow_tf32": torch.backends.cuda.matmul.allow_tf32}
    with torch.no_grad():
        enc = {"own_bf16": time_ms(lambda: model.encode(x), args.iters, args.warmup)}
        mean_own = model.encode(x).latent_dist.mean.float()
        unet_sd.USE_CONV_KERNEL = False
        try:
            enc["cudnn_bf16"] = time_ms(lambda: model.encode(x), args.iters, args.warmup)
            mean_lib = model.encode(x).latent_dist.mean.float()
        finally:
            unet_sd.USE_CONV_KERNEL = True
        m32 = AutoencoderKL(with_encoder=True).eval().to("cuda")
        m32.load_state_dict({k: v.float() for k, v in model.state_dict().items()})
        enc["cudnn_fp32"] = time_ms(lambda: m32.encode(x), args.iters, args.warmup)
        mean_32 = m32.encode(x).latent_dist.mean
        del m32
        res["encode"] = {k: _median(v) for k, v in enc.items()}
        scale = mean_32.abs().max()
        res["mean_err_vs_fp32"] = {"own_bf16_max_rel": float((mean_own - mean_32).abs().max() / scale),
                                   "cudnn_bf16_max_rel": float((mean_lib - mean_32).abs().max() / scale)}

        rows = []
        for C, H in ((128, 512), (256, 256), (512, 128)):            # the three downsamplers, eight images
            xd = torch.randn((args.batch, C, H, H), device="cuda", dtype=torch.bfloat16).contiguous(memory_format=CL)
            w = (torch.randn((C, C, 3, 3), device="cuda") / (C * 9) ** 0.5).to(torch.bfloat16)
            bias = torch.zeros(C, device="cuda", dtype=torch.bfloat16)
            wk, wcl = w.permute(0, 2, 3, 1).contiguous(), w.contiguous(memory_format=CL)
            flop = 2.0 * args.batch * (H // 2) ** 2 * C * C * 9
            own_ms = kernel_ms(lambda: ops.conv2d_down2x(xd, wk, bias))
            lib_ms = kernel_ms(lambda: F.conv2d(F.pad(xd, (0, 1, 0, 1)), wcl, bias, stride=2))
            rows.append({"C": C, "H": H, "own_ms": own_ms, "own_tflops": flop / own_ms / 1e9,
                         "pad_cudnn_ms": lib_ms, "pad_cudnn_tflops": flop / lib_ms / 1e9})
            del xd, w, wk, wcl
        res["down2x"] = rows
        conv_in = model.encoder.conv_in
        xin = x.to(torch.bfloat16).contiguous(memory_format=CL)
        res["conv_in_cudnn_ms"] = kernel_ms(lambda: conv_in(xin))
        del model

        torch.manual_seed(1)
        dec = ImageDecoder(perceiver_config=dict(num_queries=77, hidden_size=1024, encoder_hidden_size=5120,
                                                 cross_attention_frequency=1, num_hidden_layers=1, num_attention_heads=16),
                           seq_len=77, embed_dim=1024, image_size=512, vae={"with_encoder": True}).eval()
        dec = dec.to("cuda", torch.bfloat16)
        dec.decoder.unet.to(memory_format=CL)
        B = args.batch
        images = torch.rand((B, 3, 512, 512), device="cuda")
        ctx = torch.randn((B, 40, 5120), device="cuda", dtype=torch.bfloat16)
        ctx_mask = torch.ones((B, 40), dtype=torch.long, device="cuda")
        feats = [torch.randn((B, 1, 1024, s, s), device="cuda", dtype=torch.bfloat16) for s in (64, 32, 16, 8)]
        fmask = torch.ones((B, 1), dtype=torch.long, device="cuda")
        step = lambda: dec(images, ctx, ctx_mask, mmfs_features=feats, mmfs_mask=fmask,
                           generator=torch.Generator(device="cuda").manual_seed(0))
        res["image_decoder_forward"] = _median(time_ms(step, args.iters, args.warmup))
        res["image_decoder_forward"]["loss"] = float(step())

    print(f"encode of ({args.batch}, 3, 512, 512) images, median of {args.iters}:")
    for name, d in res["encode"].items():
        print(f"  {name:11s} {d['median_ms']:9.2f} ms  (min {d['min_ms']:.2f}, max {d['max_ms']:.2f})")
    print(f"  posterior mean max |err| / max|fp32|: own bf16 {res['mean_err_vs_fp32']['own_bf16_max_rel']:.3e}, "
          f"cuDNN bf16 {res['mean_err_vs_fp32']['cudnn_bf16_max_rel']:.3e}")
    print("downsample (one-sided pad + 3x3 / stride 2), one launch:")
    for r in rows:
        print(f"  {r['C']:4d}ch {r['H']}^2 -> {r['H'] // 2}^2  own {r['own_ms']:8.3f} ms {r['own_tflops']:6.1f} TF/s  "
              f"pad + cuDNN {r['pad_cudnn_ms']:8.3f} ms {r['pad_cudnn_tflops']:6.1f} TF/s")
    print(f"conv_in (3 -> 128, 512^2, cuDNN bf16): {res['conv_in_cudnn_ms']:.3f} ms")
    d = res["image_decoder_forward"]
    print(f"ImageDecoder.forward, B_I = {args.batch}: {d['median_ms']:.2f} ms (min {d['min_ms']:.2f}, max {d['max_ms']:.2f})")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--encode", action="store_true", help="time the encoder and the image-decoder loss instead")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_bench.py needs a CUDA device")
    info = gpu_info()
    print("gpu:", info)
    if args.encode:
        res = encode_bench(args, info)
        line = json.dumps(res)
        print(line)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "vae_bench_encode.json"), "w") as f:
                f.write(line + "\n")
        return
    torch.manual_seed(0)
    model = AutoencoderKL().eval().to("cuda", torch.bfloat16).to(memory_format=CL)
    z = torch.randn((args.batch, 4, 64, 64), device="cuda") * 4

    res = {"gpu": info, "batch": args.batch, "iters": args.iters,
           "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "matmul_allow_tf32": torch.backends.cuda.matmul.allow_tf32}
    with torch.no_grad():
        shapes = conv_shapes(model, z)
        decode = {}
        own = time_ms(lambda: model.decode(z), args.iters, args.warmup)
        unet_sd.USE_CONV_KERNEL = False
        try:
            cudnn = time_ms(lambda: model.decode(z), args.iters, args.warmup)
        finally:
            unet_sd.USE_CONV_KERNEL = True
        out_own = model.decode(z).float()
        unet_sd.USE_CONV_KERNEL = False
        try:
            out_lib = model.decode(z).float()
        finally:
            unet_sd.USE_CONV_KERNEL = True
        m32 = AutoencoderKL().eval().to("cuda").to(memory_format=CL)
        m32.load_state_dict({k: v.float() for k, v in model.state_dict().items()})
        fp32 = time_ms(lambda: m32.decode(z), args.iters, args.warmup)
        out_32 = m32.decode(z)
        del m32
        for name, t in (("own_bf16", own), ("cudnn_bf16", cudnn), ("cudnn_fp32", fp32)):
            decode[name] = {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t)}
        scale = out_32.abs().max()
        res["decode"] = decode
        res["err_vs_fp32"] = {"own_bf16_max_rel": float((out_own - out_32).abs().max() / scale),
                              "cudnn_bf16_max_rel": float((out_lib - out_32).abs().max() / scale)}

        rows = []
        total_own = total_lib = 0.0
        for (kind, B, Cin, Cout, H, W, k), n in sorted(shapes.items(), key=lambda kv: kv[0][4] * kv[0][5]):
            x = torch.randn((B, Cin, H, W), device="cuda", dtype=torch.bfloat16).contiguous(memory_format=CL)
            w = (torch.randn((Cout, Cin, k, k), device="cuda") / (Cin * k * k) ** 0.5).to(torch.bfloat16)
            bias = torch.zeros(Cout, device="cuda", dtype=torch.bfloat16)
            wcl = w.contiguous(memory_format=CL)
            row = {"kind": kind, "B": B, "Cin": Cin, "Cout": Cout, "H": H, "W": W, "k": k, "count": n}
            if kind == "up2x":
                Ho, Wo = 2 * H, 2 * W
                flop4 = 2.0 * B * Ho * Wo * Cout * Cin * 4
                flop9 = 2.0 * B * Ho * Wo * Cout * Cin * 9
                row["own"] = ops.conv2d_up2x_supported(x, w)
                if row["own"]:
                    wp = ops.fold_up2x_weights(w)
                    row["own_ms"] = kernel_ms(lambda: ops.conv2d_up2x(x, wp, bias))
                row["cudnn_ms"] = kernel_ms(lambda: F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), wcl, bias, padding=1))
                row["gflop_own"], row["gflop_9tap"] = flop4 / 1e9, flop9 / 1e9
                if row["own"]:
                    row["own_tflops"] = flop4 / row["own_ms"] / 1e9
                    row["own_tflops_9tap_equiv"] = flop9 / row["own_ms"] / 1e9
                row["cudnn_tflops_9tap"] = flop9 / row["cudnn_ms"] / 1e9
            else:
                flop = 2.0 * B * H * W * Cout * Cin * k * k
                row["own"] = ops.conv2d_supported(x, w, 1, k // 2)
                if row["own"]:
                    wk = w.permute(0, 2, 3, 1).contiguous()
                    row["own_ms"] = kernel_ms(lambda: ops.conv2d(x, wk, bias, 1, k // 2))
                row["cudnn_ms"] = kernel_ms(lambda: F.conv2d(x, wcl, bias, 1, k // 2))
                row["gflop"] = flop / 1e9
                if row["own"]:
                    row["own_tflops"] = flop / row["own_ms"] / 1e9
                row["cudnn_tflops"] = flop / row["cudnn_ms"] / 1e9
            total_own += n * row.get("own_ms", row["cudnn_ms"])
            total_lib += n * row["cudnn_ms"]
            rows.append(row)
            del x, w, wcl
        res["convs"] = rows
        res["convs_total_ms"] = {"own": total_own, "cudnn": total_lib}

    print(f"decode of ({args.batch}, 4, 64, 64) latents, median of {args.iters}:")
    for name, d in decode.items():
        print(f"  {name:11s} {d['median_ms']:9.2f} ms  (min {d['min_ms']:.2f}, max {d['max_ms']:.2f})")
    print(f"  max |err| / max|fp32|: own bf16 {res['err_vs_fp32']['own_bf16_max_rel']:.3e}, "
          f"cuDNN bf16 {res['err_vs_fp32']['cudnn_bf16_max_rel']:.3e}")
    print("per convolution shape (one launch; count = layers of that shape):")
    for r in rows:
        tag = f"{r['kind']:4s} B{r['B']} {r['Cin']:4d}->{r['Cout']:4d} k{r['k']} {r['H']}x{r['W']} x{r['count']}"
        own_s = f"own {r['own_ms']:8.3f} ms {r['own_tflops']:6.1f} TF/s" if r["own"] else "own  (not taken)"
        lib_tf = r.get("cudnn_tflops", r.get("cudnn_tflops_9tap"))
        extra = f"  [9-tap equiv {r['own_tflops_9tap_equiv']:.1f} TF/s]" if r["kind"] == "up2x" and r["own"] else ""
        print(f"  {tag:40s} {own_s}  cuDNN {r['cudnn_ms']:8.3f} ms {lib_tf:6.1f} TF/s{extra}")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "vae_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
