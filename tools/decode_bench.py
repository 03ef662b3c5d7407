"""Greedy decode timing of the Llama-13B MMFS decoder (random weights, bf16): prefill on B x 2048-token 4-image
sequences, then N new tokens with (a) the eager loop over the pre-allocated in-place KV cache, (b) the CUDA-graphed
decode step (InterleavedForward.enable_decode_graphs) and (c) the reference-style cat-per-token cache.
Weight-read floor per token: 13.0 B parameters x 2 B / peak HBM GB/s (workloads.measured_peaks).  Prints one JSON object."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchmarks import workloads  # noqa: E402
from mm_interleaved_b200.mm_interleaved import InterleavedForward  # noqa: E402

B = int(os.environ.get("LOCAL_BATCH", 4))
n_new = int(os.environ.get("N_NEW", 32))
wl = workloads.InterleavedCfg3(0, 1, B)
wl.make_host_inputs(pin=False)
model = workloads.full_model(with_image_decoder=False)
ids, img, nimg = (t.cuda() for t in wl.host)
rows = {}
with torch.no_grad():
    vis = model._tokenize(img)
    gen = lambda n, **kw: InterleavedForward.generate_texts(model, ids, vis, nimg, wl.N_IMG, max_new_tokens=n, eos_token_id=None, **kw)

    def per_token(**kw):
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
peaks = workloads.measured_peaks()
wbytes = 2.0 * sum(p.numel() for n, p in model.named_parameters() if n.startswith(("mm_decoder.", "text_decoder.")))
kv = 2.0 * 40 * 2 * wl.T * 5120 * B
rows.update(batch=B, context_tokens=wl.T, new_tokens=n_new, weight_bytes=wbytes, kv_bytes=kv,
            floor_ms_per_token=1e3 * (wbytes + kv) / (peaks["hbm_gbs"] * 1e9),
            graphed_frac_of_hbm_peak=(wbytes + kv) / t_graph / 1e9 / peaks["hbm_gbs"],
            tokens_per_s_graphed=B / t_graph)
print(json.dumps(rows))
