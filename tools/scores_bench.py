"""``generate_scores`` with and without ``enable_shared_context_scores`` on the Llama-13B MMFS model (random weights,
bf16, ``benchmarks.workloads.full_model``) at a VisDial-shaped workload: 4 dialogs, each a 200-token context (bos, soi,
64 image tokens, text) with 100 answer options of 2-16 tokens padded to 16.

  1. ms per dialog for both paths, alternated in one process, the best of ``--repeats`` calls each; the decoder
     positions per dialog from the shapes (default: 100 * (C + L); shared: C + 100 * (L - 1)); the peak memory torch
     allocated during each path's call above what was allocated before it (GB, 2^30 bytes); the largest |score
     difference| between the paths and whether each dialog ranks its options the same;
  2. one layer's attention (40 x 128 heads, context 200, 100 options of 16) replayed from a CUDA graph:
     ``ops.attention_prefix_shared`` against ``ops.attention`` over the replicated (100, 216) cache with past = 200.
Prints one JSON object with the card name and its power limit, read in the same run.

    python tools/scores_bench.py [--repeats 2] [--skip-model]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchmarks import workloads  # noqa: E402
from mm_interleaved_b200 import ops  # noqa: E402
from tools.kv_fp8_bench import card, graph_us  # noqa: E402

N_DIALOG, C, G, L, N_IMG_TOK = 4, 200, 100, 16, 64
HEADS, HD = 40, 128


def attention_row():
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *shape: torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    q, k, v = rnd(1, G * L, HEADS, HD), rnd(1, G * L, HEADS, HD), rnd(1, G * L, HEADS, HD)
    kp, vp = rnd(1, C, HEADS, HD), rnd(1, C, HEADS, HD)
    kr = torch.cat((kp.expand(G, -1, -1, -1), k.view(G, L, HEADS, HD)), 1).contiguous()
    vr = torch.cat((vp.expand(G, -1, -1, -1), v.view(G, L, HEADS, HD)), 1).contiguous()
    qr = q.view(G, L, HEADS, HD)
    shared = graph_us(lambda: ops.attention_prefix_shared(q, kp, vp, k, v, L))
    replicated = graph_us(lambda: ops.attention(qr, kr, vr, causal=True, past=C))
    a = ops.attention_prefix_shared(q, kp, vp, k, v, L).float().view(G, L, -1)
    b = ops.attention(qr, kr, vr, causal=True, past=C).float()
    return {"shape": f"H={HEADS} hd={HD} Tp={C} G={G} L={L}", "prefix_shared_us": round(shared, 1),
            "replicated_us": round(replicated, 1), "max_abs_diff": float((a - b).abs().max())}


def batch():
    g = torch.Generator().manual_seed(3)
    ctx = []
    for _ in range(N_DIALOG):
        t = torch.randint(3, 31000, (C,), generator=g)
        t[0], t[1] = workloads.BOS_ID, workloads.SOI_ID
        t[2:2 + N_IMG_TOK] = workloads.IMG_ID
        ctx.append(t.cuda())
    n = torch.randint(2, L + 1, (N_DIALOG, G), generator=g)
    opts = [torch.randint(3, 31000, (G, L), generator=g).cuda() for _ in range(N_DIALOG)]
    masks = [(torch.arange(L)[None, :] < n[i][:, None]).long().cuda() for i in range(N_DIALOG)]
    images = torch.rand((N_DIALOG, 3, 224, 224), generator=g).cuda().to(torch.bfloat16)
    return dict(text_ids=ctx, image_tensors=images, num_image_per_seq=torch.ones((N_DIALOG, 1), dtype=torch.long).cuda(),
                attention_mask=[torch.ones_like(t) for t in ctx], options_ids=opts, options_attn_masks=masks)


def model_rows(repeats):
    model = workloads.full_model(with_image_decoder=False)
    inputs = batch()
    best, peak, scores = {}, {}, {}
    for r in range(repeats + 1):                       # the first round warms up both paths
        for shared in (False, True):
            model.enable_shared_context_scores(shared)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            s = model.generate(mode="generate_scores", **inputs)["scores"]
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) * 1e3 / N_DIALOG
            if r > 0:
                best[shared] = min(best.get(shared, float("inf")), dt)
            peak[shared] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
            scores[shared] = s.float()
    model.enable_shared_context_scores(False)
    a, b = scores[False][:, 0], scores[True][:, 0]
    return {"dialogs": N_DIALOG, "context": C, "options": G, "option_len": L,
            "ms_per_dialog": {"default": round(best[False], 1), "shared_context": round(best[True], 1)},
            "decoder_positions_per_dialog": {"default": G * (C + L), "shared_context": C + G * (L - 1)},
            "peak_alloc_gb": {"default": round(peak[False], 2), "shared_context": round(peak[True], 2)},
            "max_abs_score_diff": float((a - b).abs().max()),
            "rankings_agree": [bool(torch.equal(a[i].argsort(descending=True), b[i].argsort(descending=True)))
                               for i in range(N_DIALOG)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scores_bench.py measures on the GPU; no CUDA device is visible")
    out = dict(card(), attention=attention_row())
    if not args.skip_model:
        with torch.no_grad():
            out["generate_scores"] = model_rows(args.repeats)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
