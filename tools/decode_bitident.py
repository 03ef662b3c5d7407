"""Bit-identity of decode attention and text generation between two trees of the project (e.g. a change and its
parent): run the same seeded cases under each tree, saving the outputs, then compare them with ``torch.equal``.

  - ops.attention (decode branch), ops.attention_decode_shared, ops.attention_decode_fp8 and
    ops.attention_decode_shared_fp8 at hd 64 / 96 / 128 / 256 in fp32 / bf16 / fp16, at one split and at many, with and
    without a key mask (one row fully masked), with past at and below the last key, shared at G = 1 and 5;
  - the tiny decoder's greedy and 3-beam ids, eager and graphed, with 16-bit and FP8 caches.

    python tools/decode_bitident.py --tree <tree> --save a.pt     (once per tree)
    python tools/decode_bitident.py --compare a.pt b.pt
"""
import argparse
import os
import sys

import torch


def op_cases(ops):
    out = {}
    H, max_new = 3, 8
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        for hd in (64, 96, 128, 256):
            for Tkv in (200, 1500):
                g = torch.Generator(device="cuda").manual_seed(hd * 7 + Tkv)
                rnd = lambda *s: torch.randn(s, device="cuda", generator=g).to(dtype)
                for G in (1, 5):
                    P = 2
                    R = P * G
                    q = rnd(R, 1, 3, H, hd)[:, :, 0]                       # a strided q, as the QKV GEMM leaves it
                    Tp = Tkv - max_new
                    kp, vp, kg, vg = rnd(P, Tp, H, hd), rnd(P, Tp, H, hd), rnd(R, max_new, H, hd), rnd(R, max_new, H, hd)
                    plen = torch.tensor([Tp - 3], device="cuda")
                    rep = lambda p, gen: torch.cat([p.repeat_interleave(G, 0)[:, :Tp - 3], gen, gen[:, -1:].expand(
                        R, 3, H, hd)], 1).contiguous()
                    k, v = rep(kp, kg), rep(vp, vg)
                    mask = (torch.rand((R, Tkv), device="cuda", generator=g) > 0.3).to(torch.uint8)
                    mask[0] = 0                                              # a fully masked row
                    q8 = [ops.quantize_kv_fp8(t) for t in (kp, vp, kg, vg, k, v)]
                    for km_name, km in (("nomask", None), ("mask", mask)):
                        for past in (Tkv - 1, Tkv // 2):
                            key = f"{dtype}_hd{hd}_T{Tkv}_G{G}_{km_name}_past{past}"
                            out[f"dense_{key}"] = ops.attention(q, k, v, key_mask=km, past=past)
                            out[f"shared_{key}"] = ops.attention_decode_shared(q, kp, vp, kg, vg, plen, key_mask=km,
                                                                               past=past)
                            (k8, ks), (v8, vs) = q8[4], q8[5]
                            out[f"fp8_{key}"] = ops.attention_decode_fp8(q, k8, v8, ks, vs, key_mask=km, past=past)
                            (kp8, ksp), (vp8, vsp), (kg8, ksg), (vg8, vsg) = q8[:4]
                            out[f"fp8shared_{key}"] = ops.attention_decode_shared_fp8(
                                q, kp8, vp8, ksp, vsp, kg8, vg8, ksg, vsg, plen, key_mask=km, past=past)
    return {k: t.cpu() for k, t in out.items()}


def generation_cases(tiny):
    out = {}
    for fp8 in (False, True):
        for nb in (1, 3):
            dev, ids, nimg, vis_d = tiny()
            dev.enable_fp8_kv_cache(fp8)
            kw = dict(max_new_tokens=7, eos_token_id=[2, 17], min_length=3, num_beams=nb)
            out[f"gen_fp8{fp8}_nb{nb}_eager"] = dev.generate_texts(ids, vis_d, nimg, 2, **kw).cpu()
            dev.enable_decode_graphs()
            out[f"gen_fp8{fp8}_nb{nb}_graphed"] = dev.generate_texts(ids, vis_d, nimg, 2, **kw).cpu()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree")
    ap.add_argument("--save")
    ap.add_argument("--compare", nargs=2)
    a = ap.parse_args()
    if a.compare:
        x, y = (torch.load(p) for p in a.compare)
        assert x.keys() == y.keys(), set(x) ^ set(y)
        bad = [k for k in x if not (x[k].shape == y[k].shape and torch.equal(x[k], y[k]))]
        print(f"{len(x)} outputs compared, {len(bad)} differ{': ' + ', '.join(bad[:20]) if bad else ''}")
        sys.exit(1 if bad else 0)
    if not torch.cuda.is_available():
        raise SystemExit("decode_bitident needs a CUDA device")
    sys.path.insert(0, os.path.abspath(a.tree))
    from mm_interleaved_b200 import ops
    from tests.test_kv_fp8_gpu import _tiny
    with torch.no_grad():
        out = op_cases(ops)
        out.update(generation_cases(_tiny))
    torch.save(out, a.save)
    print(f"{len(out)} outputs saved from {ops.__file__}")


if __name__ == "__main__":
    main()
