"""Decode timing of the Llama-13B MMFS decoder (random weights, bf16): prefill on B x 2048-token 4-image sequences,
then N new tokens with (a) the eager loop over the pre-allocated in-place KV cache (``generation.token_loop``), (b) the
CUDA-graphed decode step (InterleavedForward.enable_decode_graphs: ``generation.TokenDecoder``, whose token choice is
one ``ops.decode_select`` launch) and (c) the reference-style cat-per-token cache, greedy.
Weight-read floor per token: 13.0 B parameters x 2 B / peak HBM GB/s (workloads.measured_peaks).

Then the reference's release inference settings (mm_inference.yaml: top_p 0.9, temperature 1.0, repetition penalty
1.3, min_length 8, 90 new tokens; eos_token_id=None so every step decodes a real token), eager against graphed, for
greedy + penalty and for sampling (``release_*`` rows), and the token choice alone: ``ops.decode_select`` against the
torch chain of the eager loop it replaces (gather / scatter penalty, sort, softmax, cumsum, masked fill, multinomial;
``select_*`` rows) at B in {1, 4, 8}, V = 32002, CUDA events over many launches.  Prints one JSON object with the card
name, its power limit and SM clock read in the same run.

    LOCAL_BATCH=4 N_NEW=32 python tools/decode_bench.py         # SELECT_ONLY=1: only the token-choice rows
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

B = int(os.environ.get("LOCAL_BATCH", 4))
n_new = int(os.environ.get("N_NEW", 32))
RELEASE = dict(top_p=0.9, temperature=1.0, repetition_penalty=1.3, min_length=8)
RELEASE_NEW = 90
V = 32002


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        out = []
    row = out[torch.cuda.current_device()] if len(out) > torch.cuda.current_device() else ""
    return {"card": torch.cuda.get_device_name(), "nvidia_smi": dict(zip(q.split(","), [s.strip() for s in row.split(",")]))}


def torch_chain(scores, prev, sample, gen):
    """The eager loop's token choice (generation.token_loop) at the release settings."""
    p, T, top_p = RELEASE["repetition_penalty"], RELEASE["temperature"], RELEASE["top_p"]
    picked = scores.gather(1, prev)
    scores = scores.scatter(1, prev, torch.where(picked < 0, picked * p, picked / p))
    if not sample:
        return scores.argmax(-1)
    scores = scores / T
    srt, idx = scores.sort(dim=-1, descending=False)
    drop = srt.softmax(-1).cumsum(-1) <= (1.0 - top_p)
    drop[:, -1] = False
    scores = scores.masked_fill(drop.scatter(1, idx, drop), float("-inf"))
    return torch.multinomial(scores.softmax(-1), 1, generator=gen).squeeze(1)


def select_rows(rows, iters=500):
    """us per call of decode_select and of the torch chain, CUDA events around `iters` back-to-back calls."""
    g = torch.Generator(device="cuda").manual_seed(0)
    for b in (1, 4, 8):
        logits = torch.randn((b, V), device="cuda", generator=g) * 3
        hist = torch.randint(0, V, (b, RELEASE_NEW), device="cuda", generator=g)
        step = torch.tensor([RELEASE_NEW // 2], device="cuda")
        prev = hist[:, :RELEASE_NEW // 2].contiguous()
        fin = torch.zeros(b, dtype=torch.bool, device="cuda")
        nxt = torch.zeros((b, 1), dtype=torch.long, device="cuda")
        params = torch.tensor([RELEASE["repetition_penalty"], RELEASE["temperature"], RELEASE["top_p"]], device="cuda")
        seed = torch.tensor([7], device="cuda")
        for sample in (False, True):
            name = "sample" if sample else "greedy_penalty"
            runs = {"decode_select": lambda: ops.decode_select(logits, hist, step, fin, nxt, params, pad_id=0, min_length=8,
                                                               sample=sample, seed=seed),
                    "torch_chain": lambda: torch_chain(logits, prev, sample, g)}
            for what, fn in runs.items():
                for _ in range(20):
                    fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                rows[f"select_{name}_B{b}_{what}_us"] = 1e3 * e0.elapsed_time(e1) / iters
            # the kernel without the Python launch path: 50 launches captured in one graph, replayed
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(50):
                    runs["decode_select"]()
            graph.replay()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(iters // 50):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            rows[f"select_{name}_B{b}_decode_select_in_graph_us"] = 1e3 * e0.elapsed_time(e1) / (iters // 50 * 50)


rows = card()
select_rows(rows)
if os.environ.get("SELECT_ONLY"):
    print(json.dumps(rows))
    sys.exit(0)

wl = workloads.InterleavedCfg3(0, 1, B)
wl.make_host_inputs(pin=False)
model = workloads.full_model(with_image_decoder=False)
ids, img, nimg = (t.cuda() for t in wl.host)
with torch.no_grad():
    vis = model._tokenize(img)
    gen = lambda n, **kw: InterleavedForward.generate_texts(model, ids, vis, nimg, wl.N_IMG, max_new_tokens=n, eos_token_id=None, **kw)

    def per_token(n_new=n_new, **kw):
        """(time of 1 + n_new tokens - time of 1 token) / n_new, each the best of 3 runs (the first run of a shape pays
        allocations / graph capture)."""
        t1 = tn = None
        for rep in range(3):
            torch.cuda.synchronize(); t0 = time.time()
            gen(1, **kw)
            torch.cuda.synchronize(); ta = time.time()
            out = gen(1 + n_new, **kw)
            torch.cuda.synchronize(); tb = time.time()
            t1 = (ta - t0) if t1 is None else min(t1, ta - t0)
            tn = (tb - ta) if tn is None else min(tn, tb - ta)
        return (tn - t1) / n_new, 1e3 * t1, out

    t_eager, pre, out_e = per_token(static_cache=True)
    rows["eager_static_cache_ms_per_token"] = 1e3 * t_eager
    rows["prefill_plus_1_ms"] = pre
    model.enable_decode_graphs(True)
    t_graph, _, out_g = per_token(static_cache=True)
    model.enable_decode_graphs(False)
    rows["graphed_ms_per_token"] = 1e3 * t_graph
    rows["graph_tokens_equal_eager"] = bool(torch.equal(out_e, out_g))
    t_cat, _, _ = per_token(static_cache=False)
    rows["cat_cache_ms_per_token"] = 1e3 * t_cat

    pen = dict(repetition_penalty=RELEASE["repetition_penalty"], min_length=RELEASE["min_length"])
    smp = dict(RELEASE, use_nucleus_sampling=True)
    t_e, _, out_e = per_token(RELEASE_NEW, **pen)
    rows["release_greedy_penalty_eager_ms_per_token"] = 1e3 * t_e
    t_s, _, _ = per_token(RELEASE_NEW, **smp)
    rows["release_sample_eager_ms_per_token"] = 1e3 * t_s
    model.enable_decode_graphs(True, sampling=True)
    t_g, _, out_g = per_token(RELEASE_NEW, **pen)
    rows["release_greedy_penalty_graphed_ms_per_token"] = 1e3 * t_g
    rows["release_greedy_penalty_tokens_equal_eager"] = bool(torch.equal(out_e, out_g))
    t_gs, _, out_s = per_token(RELEASE_NEW, **smp)
    rows["release_sample_graphed_ms_per_token"] = 1e3 * t_gs
    rows["release_sample_ids_in_vocab"] = bool(int(out_s.min()) >= 0 and int(out_s.max()) < V)
    model.enable_decode_graphs(False)
peaks = workloads.measured_peaks()
wbytes = 2.0 * sum(p.numel() for n, p in model.named_parameters() if n.startswith(("mm_decoder.", "text_decoder.")))
kv = 2.0 * 40 * 2 * wl.T * 5120 * B
rows.update(batch=B, context_tokens=wl.T, new_tokens=n_new, release_new_tokens=RELEASE_NEW, weight_bytes=wbytes, kv_bytes=kv,
            floor_ms_per_token=1e3 * (wbytes + kv) / (peaks["hbm_gbs"] * 1e9),
            graphed_frac_of_hbm_peak=(wbytes + kv) / t_graph / 1e9 / peaks["hbm_gbs"],
            tokens_per_s_graphed=B / t_graph)
rows.update(card())
print(json.dumps(rows))
