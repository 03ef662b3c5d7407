"""Beam-search timing of the Llama-13B MMFS decoder (random weights, bf16): 5 beams, eos [eos, soi], min_length 8,
20 new tokens, the eager beam loop (``generation.beam_search``) against the graphed beam step (``enable_decode_graphs``:
``generation.BeamDecoder``, ``ops.beam_select`` + ``ops.kv_beam_reorder`` + the decoder in one graph replay), on two
prompt shapes:
  caption: 1 image (64 image tokens) in an 80-token prompt, the reference's captioning setting, B in {1, 4};
  long:    the 2048-token 4-image prompt of tools/decode_bench.py, B in {1, 2, 4}.  At B = 4 only the graphed loops run:
           the eager loop's 20 beam rows each hold a copy of the prompt's cache, 34 GB next to the 26 GB of weights and
           their ~18 GB of fused copies, more than an 80 GB card holds.  The graphed decoder stores the prompt once per
           prompt (7.5 GB at B = 4).
The same for beam sample (``use_nucleus_sampling=True``, top_p 0.9, temperature 1: the same eager loop with ``sample`` against
the graphed ``ops.beam_sample`` step under ``enable_decode_graphs(True, sampling=True)``; their draws differ by design,
so those ids are not compared).  With random weights eos is practically never chosen, so every step decodes.  ms per
token = (time of a 20-token call - time of a 1-token call) / 19, each the best of 2 runs; the ids of the eager and
graphed beam searches are compared.  Beside each ms per token: the peak memory allocated by torch during the 20-token
calls, the model's weights included (GB, 2^30 bytes).  Then the kernels alone (beam_select, beam_sample, the cache
reorder) at the step in the middle of a run (step 10), CUDA events over many launches, and one layer's decode attention
of that step, replayed from a CUDA graph, over the replicated cache (``ops.attention``) and over the shared prefix
(``ops.attention_decode_shared``).
Prints one JSON object with the card name, its power limit and SM clock read in the same run.

    python tools/beam_bench.py
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

NB, MAX_NEW, MIN_LEN, V = 5, 20, 8, 32002
LAYERS, HIDDEN, HEADS = 40, 5120, 40


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
    for _ in range(10):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / iters


def graph_timed(fn, per_graph=20, iters=20):
    """us per call of ``fn`` replayed from a CUDA graph of ``per_graph`` calls: the device time of a graphed step's
    kernels, without the Python enqueue cost that ``timed`` includes."""
    fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(per_graph):
            fn()
    return timed(graph.replay, iters) / per_graph


def kernel_rows(rows, step=MAX_NEW // 2):
    g = torch.Generator(device="cuda").manual_seed(0)
    eos = torch.tensor([2, 32000], device="cuda")
    for B in (1, 4):
        R = B * NB
        logits = torch.randn((R, V), device="cuda", generator=g) * 3
        st = torch.tensor([step], device="cuda")
        bufs = dict(params=torch.tensor([1.0, 1.0], dtype=torch.float64, device="cuda"),
                    beam_scores=torch.randn(R, device="cuda", generator=g) - 10,
                    history=torch.randint(0, V, (R, MAX_NEW), device="cuda", generator=g),
                    next_ids=torch.zeros((R, 1), dtype=torch.long, device="cuda"),
                    parent=torch.zeros(R, dtype=torch.long, device="cuda"),
                    done=torch.zeros(B, dtype=torch.bool, device="cuda"),
                    hyp_scores=torch.zeros((B, NB), dtype=torch.float64, device="cuda"),
                    hyp_ids=torch.zeros((B, NB, MAX_NEW), dtype=torch.long, device="cuda"),
                    hyp_meta=torch.full((B, NB, 2), -1, dtype=torch.long, device="cuda"),
                    scratch=torch.zeros(R * ops.beam_candidates(NB, 2), dtype=torch.long, device="cuda"))
        rows[f"beam_select_B{B}_us"] = timed(lambda: ops.beam_select(logits, st, num_beams=NB, eos=eos, min_length=MIN_LEN,
                                                                      **bufs), 200)
        sbufs = dict(bufs, params=torch.tensor([1.0, 1.0, 1.0, 0.9], dtype=torch.float64, device="cuda"),
                     scratch=torch.zeros(ops.beam_sample_scratch(NB, R), dtype=torch.long, device="cuda"),
                     error=torch.zeros(1, dtype=torch.int32, device="cuda"), seed=torch.tensor([5], device="cuda"))
        rows[f"beam_sample_B{B}_us"] = timed(lambda: ops.beam_sample(logits, st, num_beams=NB, eos=eos, min_length=MIN_LEN,
                                                                      **sbufs), 200)
        # the cache reorder at 13B widths, every row moved (cyclic parents), prompt of 2048 tokens
        T = 2048 + MAX_NEW
        kv = torch.zeros((2 * LAYERS, R, T, HEADS, HIDDEN // HEADS), dtype=torch.bfloat16, device="cuda")
        parent = torch.tensor([b * NB + (j + 1) % NB for b in range(B) for j in range(NB)], device="cuda")
        cur = torch.tensor([2048 + step], device="cuda")
        rows[f"kv_beam_reorder_B{B}_us"] = timed(lambda: ops.kv_beam_reorder(kv, parent, cur, st, NB, MAX_NEW), 100)
        rows[f"kv_beam_reorder_B{B}_bytes"] = 2 * 2 * LAYERS * R * step * HIDDEN * 2          # read + write, K and V
        del kv
        torch.cuda.empty_cache()
        # one layer's decode attention of the graphed step, replayed from a graph: over the replicated cache
        # (ops.attention, the layout before the shared prefix) and over the shared prefix (ops.attention_decode_shared)
        hd = HIDDEN // HEADS
        for name, L in (("caption", 80), ("long", 2048)):
            t_max = (L + MAX_NEW + 255) // 256 * 256
            rnd = lambda *shape: torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
            q = rnd(R, 1, 3, HEADS, hd)[:, :, 0]
            kr, vr = rnd(R, t_max, HEADS, hd), rnd(R, t_max, HEADS, hd)
            kp, vp = kr[::NB, :t_max - MAX_NEW].contiguous(), vr[::NB, :t_max - MAX_NEW].contiguous()
            kg, vg = kr[:, L:L + MAX_NEW].contiguous(), vr[:, L:L + MAX_NEW].contiguous()
            mask = torch.zeros((R, t_max), dtype=torch.uint8, device="cuda")
            mask[:, :L + step + 1] = 1
            plen = torch.tensor([L], device="cuda")
            rep_us = graph_timed(lambda: ops.attention(q, kr, vr, key_mask=mask, past=t_max - 1))
            sh_us = graph_timed(lambda: ops.attention_decode_shared(q, kp, vp, kg, vg, plen, key_mask=mask, past=t_max - 1))
            rows[f"attn_decode_{name}_B{B}_replicated_us"], rows[f"attn_decode_{name}_B{B}_shared_us"] = rep_us, sh_us
            del kr, vr, kp, vp, kg, vg


def caption_inputs(B):
    """1 image (64 image tokens after <soi>) in an 80-token prompt."""
    g = torch.Generator().manual_seed(77)
    W = workloads.InterleavedCfg3
    ids = torch.randint(3, 31999, (B, 80), generator=g)
    ids[:, 0] = workloads.BOS_ID
    ids[:, 1] = W.SOI_ID
    ids[:, 2:2 + W.TOK_PER_IMG] = W.IMG_ID
    images = torch.rand((B, 3, 224, 224), generator=g)
    return ids, images, torch.ones(B, dtype=torch.long), 1


def long_inputs(B):
    wl = workloads.InterleavedCfg3(0, 1, B)
    wl.make_host_inputs(pin=False)
    ids, img, nimg = wl.host
    return ids, img, nimg, wl.N_IMG


rows = card()
kernel_rows(rows)
model = workloads.full_model(with_image_decoder=False)
eos = [2, workloads.InterleavedCfg3.SOI_ID]
with torch.no_grad():
    for shape, make, batches in (("caption", caption_inputs, (1, 4)), ("long", long_inputs, (1, 2, 4))):
        for B in batches:
            ids, img, nimg, n_img = make(B)
            ids, img, nimg = ids.cuda(), img.cuda(), nimg.cuda()
            vis = model._tokenize(img)

            def per_token(graphed, sample=False):
                """Best of 2 calls at MAX_NEW and at 1 new token (the first graphed call of a length captures its
                graph); one beam graph is alive at a time, since one cache at the long shape takes up to 19 GB."""
                gen = lambda n: InterleavedForward.generate_texts(
                    model, ids, vis, nimg, n_img, max_new_tokens=n, eos_token_id=eos, min_length=MIN_LEN, num_beams=NB,
                    use_nucleus_sampling=sample, top_p=0.9, generator=torch.Generator(device="cuda").manual_seed(0))
                best, out = {}, None
                torch.cuda.reset_peak_memory_stats()
                for n in (MAX_NEW, 1):
                    model.enable_decode_graphs(graphed, sampling=sample)
                    for _ in range(2):
                        torch.cuda.synchronize(); t0 = time.time()
                        o = gen(n)
                        torch.cuda.synchronize(); dt = time.time() - t0
                        best[n] = min(best.get(n, dt), dt)
                        out = o if n == MAX_NEW else out
                    if n == MAX_NEW:
                        peak = torch.cuda.max_memory_allocated() / 2**30
                    model.enable_decode_graphs(False)
                    torch.cuda.empty_cache()
                return 1e3 * (best[MAX_NEW] - best[1]) / (MAX_NEW - 1), out, peak

            key = f"{shape}_B{B}"
            rows[f"{key}_prompt_tokens"] = ids.shape[1]
            eager = not (shape == "long" and B == 4)                    # the eager loop's cache does not fit
            outs = {}
            for sample, name in ((False, ""), (True, "sample_")):
                for graphed in (False, True) if eager else (True,):
                    run = name + ("graphed" if graphed else "eager")
                    ms, outs[run], peak = per_token(graphed, sample=sample)
                    rows[f"{key}_{run}_ms_per_token"], rows[f"{key}_{run}_peak_gb"] = ms, peak
            if eager:
                rows[f"{key}_ids_equal"] = bool(torch.equal(outs["eager"], outs["graphed"]))
            del vis
            torch.cuda.empty_cache()
rows.update(beams=NB, new_tokens=MAX_NEW, min_length=MIN_LEN)
rows.update(card())
print(json.dumps(rows))
