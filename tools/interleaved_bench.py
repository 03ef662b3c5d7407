"""Per-turn time of ``MMInterleaved.generate_interleaved`` against the reference-style loop, at the release sizes.

    python tools/interleaved_bench.py [--reps 3] [--num-iter 4]

Model: ``benchmarks.workloads.full_model()`` (Vicuna-13B decoder with MMFS, CLIP ViT-L/14 + adapter + Q-Former
tokenizer, SD-2.1-base UNet + MMFSNet image decoder; bf16, seeded random weights) plus the SD-2.1 VAE decoder, with the
tokenizer and UNet graphs and graphed decoding on (``enable_cuda_graphs``, ``enable_decode_graphs(True,
sampling=True)``).  Sample: an 8-image context of ``--tokens`` ids (64 ``<image>`` ids per image) that the turns grow
towards the 2048-token budget; generation keywords of mm_inference.yaml (max_length 90, min_length 8, greedy
width 1, nucleus sampling with top_p 0.9, repetition penalty 1.3, guidance 7.5, 30 denoise steps, 1 image), ``num_iter``
turns from a text turn with ``force_gen_image_next`` (text, image, text, image).

The reference-style loop is inference.py's: ``model.generate(mode=...)`` per turn over the whole context, the generated
image re-entered through PIL on the host (tensor_to_pil, BOX halving, BICUBIC to 224, / 255).  The two alternate
within one run, after one warm-up run each (graph captures); every turn ends in a device synchronise.  Also timed: the
re-entry kernel alone (CUDA events over many launches) and the host PIL path it replaces.  Prints one JSON line with
the card's name and power limit, read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.workloads import BOS_ID, IMG_ID, SOI_ID, full_model  # noqa: E402

GEN = dict(max_length=90, min_length=8, num_beams=1, use_nucleus_sampling=True, top_p=0.9, repetition_penalty=1.3,
           guidance_scale=7.5, num_inference_steps=30, num_validation_images=1)       # mm_inference.yaml:49-57
N_IMG, N_TOK, R = 8, 64, 224


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
    except Exception as e:                                                   # noqa: BLE001
        name, power = torch.cuda.get_device_name(), f"unknown ({type(e).__name__})"
    return name, power


def build():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    model = full_model()
    torch.manual_seed(5)
    vae = AutoencoderKL().eval().to("cuda", torch.bfloat16).to(memory_format=torch.channels_last)
    sd = model.image_decoder.decoder
    sd.vae, sd.vae_decode = vae, vae.decode
    model.enable_cuda_graphs(tokenizer=True)
    model.enable_decode_graphs(True, sampling=True)
    return model


def sample(T):
    g = torch.Generator().manual_seed(2048)
    ids = torch.randint(3, 31999, (1, T), generator=g)
    ids[:, 0] = BOS_ID
    stride = (T - 40) // N_IMG
    for k in range(N_IMG):
        s = 8 + k * stride
        ids[:, s] = SOI_ID
        ids[:, s + 1:s + 1 + N_TOK] = IMG_ID
    images = torch.rand((N_IMG, 3, R, R), generator=g)
    return dict(text_ids=ids.cuda(), attention_mask=torch.ones_like(ids).cuda(), image_tensors=images.cuda(),
                num_image_per_seq=torch.tensor([N_IMG], device="cuda"), target_image_idxs=torch.tensor([N_IMG - 1],
                                                                                                   device="cuda"))


def pil_reentry(image):
    """update_image's host path: tensor_to_pil, center_crop_arr(224) with PIL, float32 / 255."""
    from PIL import Image
    arr = image.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8).numpy()
    pil = Image.fromarray(arr).convert("RGB")
    while min(*pil.size) >= 2 * R:
        pil = pil.resize(tuple(x // 2 for x in pil.size), resample=Image.BOX)
    scale = R / min(*pil.size)
    pil = pil.resize(tuple(round(x * scale) for x in pil.size), resample=Image.BICUBIC)
    arr = np.array(pil)
    cy, cx = (arr.shape[0] - R) // 2, (arr.shape[1] - R) // 2
    return torch.from_numpy(arr[cy:cy + R, cx:cx + R].astype(np.float32).transpose([2, 0, 1]) / 255.0)


def reference_loop(model, inputs, num_iter, seed):
    """inference.py::inference_all for one sample (generate_texts first, force_gen_image_next); per-turn seconds."""
    inputs = {k: v.clone() for k, v in inputs.items()}
    gen = torch.Generator(device="cuda").manual_seed(seed)
    mode, times = "generate_texts", []
    st = model.special_token_dict
    for _ in range(num_iter):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = model.generate(mode=mode, **inputs, generator=gen, **GEN)
        if mode == "generate_texts":
            t = out["text_ids"][0][1:]
            if t[-1] == st["eos_token_id"]:
                t = t[:-1]
            if t[-1] != st["soi_token_id"]:
                t = torch.cat((t, torch.tensor([st["soi_token_id"]]).type_as(t)))
            t = torch.cat((t, torch.tensor([st["image_token_id"]] * N_TOK).type_as(t)))
            inputs["image_tensors"] = torch.cat([inputs["image_tensors"], torch.full((1, 3, R, R), 0.5, device="cuda")])
            inputs["target_image_idxs"] = inputs["target_image_idxs"] + 1
            inputs["num_image_per_seq"] = inputs["num_image_per_seq"] + 1
            inputs["text_ids"] = torch.cat((inputs["text_ids"], t[None].cuda()), dim=-1)
            inputs["attention_mask"] = torch.cat((inputs["attention_mask"], torch.ones_like(t[None]).cuda()), dim=-1)
            mode = "generate_images"
        else:
            inputs["image_tensors"][-1, ...] = pil_reentry(out["image"][0]).cuda()
            mode = "generate_texts"
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return times, int(inputs["text_ids"].shape[1])


def session_run(model, inputs, num_iter, seed):
    """generate_interleaved with each turn timed (the session's turn methods wrapped with a synchronise on each side)."""
    from mm_interleaved_b200 import interleaved
    times = []
    cls = interleaved.InterleavedSession
    orig = cls.text_turn, cls.image_turn

    def timed(fn):
        def run(self, *a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(self, *a, **k)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            return out
        return run

    cls.text_turn, cls.image_turn = timed(orig[0]), timed(orig[1])
    try:
        out = model.generate_interleaved(**{k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors",
                                                                   "num_image_per_seq")},
                                         num_iter=num_iter, force_gen_image_next=True,
                                         generator=torch.Generator(device="cuda").manual_seed(seed), **GEN)
    finally:
        cls.text_turn, cls.image_turn = orig
    return times, int(out["text_ids"].shape[1])


def reentry_times(iters=200):
    from mm_interleaved_b200 import ops
    img = torch.rand((1, 3, 512, 512), device="cuda")
    out = torch.empty((1, 3, R, R), device="cuda")
    for _ in range(10):
        ops.image_reentry(img, R, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.image_reentry(img, R, out=out)
    e1.record()
    torch.cuda.synchronize()
    kernel_us = e0.elapsed_time(e1) * 1000.0 / iters
    host = []
    for _ in range(20):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        x = pil_reentry(img[0].clone()).cuda()
        torch.cuda.synchronize()
        host.append(time.perf_counter() - t0)
    same = torch.equal(x.view(torch.int32), out[0].view(torch.int32))
    return kernel_us, float(np.median(host)) * 1e6, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--num-iter", type=int, default=4)
    ap.add_argument("--tokens", type=int, default=1700)
    args = ap.parse_args()
    name, power = card()
    model = build()
    inputs = sample(args.tokens)
    with torch.no_grad():
        session_run(model, inputs, args.num_iter, 0)                          # warm-up: graph captures
        reference_loop(model, inputs, args.num_iter, 0)
        sess, ref = [], []
        for r in range(args.reps):                                            # alternate, order swapped per rep
            runs = [("s", session_run), ("r", reference_loop)]
            for kind, fn in (runs if r % 2 == 0 else runs[::-1]):
                t, final_len = fn(model, inputs, args.num_iter, r + 1)
                (sess if kind == "s" else ref).append(t)
        kernel_us, pil_us, same = reentry_times()
    med = lambda rows: [round(float(np.median([row[i] for row in rows])) * 1000.0, 1) for i in range(len(rows[0]))]
    s_ms, r_ms = med(sess), med(ref)
    print(json.dumps({
        "tool": "interleaved_bench", "gpu": name, "power_limit": power, "reps": args.reps,
        "initial_tokens": args.tokens, "final_tokens": final_len, "images_in": N_IMG, "num_iter": args.num_iter,
        "turns": ["text" if i % 2 == 0 else "image" for i in range(args.num_iter)],
        "session_ms_per_turn": s_ms, "reference_loop_ms_per_turn": r_ms,
        "session_ms_total": round(sum(s_ms), 1), "reference_loop_ms_total": round(sum(r_ms), 1),
        "reentry_kernel_us": round(kernel_us, 2), "reentry_host_pil_us": round(pil_us, 1),
        "reentry_bit_identical_to_pil": bool(same)}))


if __name__ == "__main__":
    main()
