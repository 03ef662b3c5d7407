"""The FP8 KV cache (``enable_fp8_kv_cache``) against the 16-bit cache on the Llama-13B MMFS decoder (random weights,
bf16):

  1. one layer's decode attention (40 x 128 heads) replayed from a CUDA graph, 16-bit (``ops.attention`` /
     ``ops.attention_decode_shared``) against FP8 (``ops.attention_decode_fp8`` / ``ops.attention_decode_shared_fp8``),
     at the caption prompt (80 tokens) and the 2048-token 4-image prompt, B in {1, 4}, over a per-row cache ("plain",
     the greedy decoder's) and over the shared prompt with 5 beams ("shared", the beam decoder's), each with the K / V
     bytes a call reads (from the shapes) and the rate that gives;
  2. graphed decoding at the 2048-token prompt: greedy (B = 1) and 5-beam search (B = 1 and 4), 20 new tokens, the two
     caches alternated in one process; ms per token = (time of a 20-token call - time of a 1-token call) / 19, each the
     best of ``--repeats`` calls; beside it the peak memory torch allocated during the first 20-token call (which
     allocates the graphed decoder and its cache) above what was allocated before it (GB, 2^30 bytes), and whether the
     two caches chose the same ids.
Prints one JSON object with the card name and its power limit, read in the same run.

    python tools/kv_fp8_bench.py [--repeats 2] [--skip-model]
"""
import argparse
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

NB, MAX_NEW, MIN_LEN = 5, 20, 8
HEADS, HD = 40, 128


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        out = []
    row = out[torch.cuda.current_device()] if len(out) > torch.cuda.current_device() else ""
    return {"card": torch.cuda.get_device_name(), "nvidia_smi": dict(zip(q.split(","), [s.strip() for s in row.split(",")]))}


def graph_us(fn, per_graph=20, iters=50):
    """us per call of ``fn``, replayed from a CUDA graph of ``per_graph`` calls (CUDA events around ``iters`` replays)."""
    fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(per_graph):
            fn()
    for _ in range(5):
        graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / (iters * per_graph)


def attention_rows(rows):
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *shape: torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    Hs = ops.kv_scale_heads(HEADS)
    for name, L in (("caption", 80), ("long", 2048)):
        t_max = (L + MAX_NEW + 255) // 256 * 256
        step = MAX_NEW // 2
        n_keys = L + step + 1
        for B in (1, 4):
            # plain: B rows, each with its own cache (the greedy decoder); every visible key is read once
            q = rnd(B, 1, 3, HEADS, HD)[:, :, 0]
            k, v = rnd(B, t_max, HEADS, HD), rnd(B, t_max, HEADS, HD)
            (k8, ks), (v8, vs) = ops.quantize_kv_fp8(k), ops.quantize_kv_fp8(v)
            ks, vs = (torch.nn.functional.pad(s, (0, Hs - HEADS)) for s in (ks, vs))
            mask = torch.zeros((B, t_max), dtype=torch.uint8, device="cuda")
            mask[:, :n_keys] = 1
            us16 = graph_us(lambda: ops.attention(q, k, v, key_mask=mask, past=t_max - 1))
            us8 = graph_us(lambda: ops.attention_decode_fp8(q, k8, v8, ks, vs, key_mask=mask, past=t_max - 1))
            b16 = 2 * B * n_keys * HEADS * HD * 2
            b8 = 2 * B * n_keys * HEADS * (HD + 4)
            key = f"attn_{name}_B{B}_plain"
            rows.update({f"{key}_16bit_us": us16, f"{key}_fp8_us": us8, f"{key}_16bit_GBps": b16 / us16 / 1e3,
                         f"{key}_fp8_GBps": b8 / us8 / 1e3})
            del k, v, k8, v8
            # shared: B prompts of NB beams each (the graphed beam search)
            R = B * NB
            q = rnd(R, 1, 3, HEADS, HD)[:, :, 0]
            kp, vp = rnd(B, t_max - MAX_NEW, HEADS, HD), rnd(B, t_max - MAX_NEW, HEADS, HD)
            kg, vg = rnd(R, MAX_NEW, HEADS, HD), rnd(R, MAX_NEW, HEADS, HD)
            (kp8, ksp), (vp8, vsp), (kg8, ksg), (vg8, vsg) = (ops.quantize_kv_fp8(t) for t in (kp, vp, kg, vg))
            ksp, vsp, ksg, vsg = (torch.nn.functional.pad(s, (0, Hs - HEADS)) for s in (ksp, vsp, ksg, vsg))
            mask = torch.zeros((R, t_max), dtype=torch.uint8, device="cuda")
            mask[:, :n_keys] = 1
            plen = torch.tensor([L], device="cuda")
            us16 = graph_us(lambda: ops.attention_decode_shared(q, kp, vp, kg, vg, plen, key_mask=mask, past=t_max - 1))
            us8 = graph_us(lambda: ops.attention_decode_shared_fp8(q, kp8, vp8, ksp, vsp, kg8, vg8, ksg, vsg, plen,
                                                                   key_mask=mask, past=t_max - 1))
            per_key = (B * L + R * (step + 1))                 # the prompt once per prompt, the generated keys per row
            key = f"attn_{name}_B{B}_shared{NB}"
            rows.update({f"{key}_16bit_us": us16, f"{key}_fp8_us": us8,
                         f"{key}_16bit_GBps": 2 * per_key * HEADS * HD * 2 / us16 / 1e3,
                         f"{key}_fp8_GBps": 2 * per_key * HEADS * (HD + 4) / us8 / 1e3})
            del kp, vp, kg, vg, kp8, vp8, kg8, vg8
            torch.cuda.empty_cache()


def model_rows(rows, repeats):
    model = workloads.full_model(with_image_decoder=False)
    model.enable_decode_graphs()
    eos = [2, workloads.InterleavedCfg3.SOI_ID]
    with torch.no_grad():
        for mode, B in (("greedy", 1), ("beam", 1), ("beam", 4)):
            wl = workloads.InterleavedCfg3(0, 1, B)
            wl.make_host_inputs(pin=False)
            ids, img, nimg = (t.cuda() for t in wl.host)
            vis = model._tokenize(img)
            nb = NB if mode == "beam" else 1
            gen = lambda n: InterleavedForward.generate_texts(model, ids, vis, nimg, wl.N_IMG, max_new_tokens=n,
                                                              eos_token_id=eos, min_length=MIN_LEN, num_beams=nb)
            best, peak, out = {}, {}, {}
            for _ in range(repeats):
                for fp8 in (False, True):                           # alternated: other work shares the host
                    model.enable_fp8_kv_cache(fp8)                  # drops the other cache's graph and buffers
                    torch.cuda.empty_cache()
                    for n in (MAX_NEW, 1):
                        torch.cuda.synchronize()
                        base = torch.cuda.memory_allocated()
                        torch.cuda.reset_peak_memory_stats()
                        gen(n)                                      # allocates this length's decoder, captures its graph
                        torch.cuda.synchronize()
                        if n == MAX_NEW:
                            peak[fp8] = (torch.cuda.max_memory_allocated() - base) / 2**30
                        t0 = time.time()
                        o = gen(n)
                        torch.cuda.synchronize()
                        dt = time.time() - t0
                        best[(fp8, n)] = min(best.get((fp8, n), dt), dt)
                        if n == MAX_NEW:
                            out[fp8] = o.cpu()
            key = f"long_{mode}_B{B}"
            rows[f"{key}_prompt_tokens"] = ids.shape[1]
            for fp8, name in ((False, "16bit"), (True, "fp8")):
                rows[f"{key}_{name}_ms_per_token"] = 1e3 * (best[(fp8, MAX_NEW)] - best[(fp8, 1)]) / (MAX_NEW - 1)
                rows[f"{key}_{name}_call_gb"] = peak[fp8]
            rows[f"{key}_ids_equal"] = bool(out[False].shape == out[True].shape and torch.equal(out[False], out[True]))
            del vis
            model.enable_fp8_kv_cache(False)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--skip-model", action="store_true", help="the attention kernels only")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_fp8_bench needs a CUDA device")
    rows = card()
    attention_rows(rows)
    if not a.skip_model:
        model_rows(rows, a.repeats)
    rows.update(beams=NB, new_tokens=MAX_NEW, min_length=MIN_LEN)
    rows.update(card())
    print(json.dumps(rows))
