"""GPU tests of ``ops.decode_select`` (csrc/decode_select_sm100.cu) and of the graphed decode step built on it:
the greedy processors bit for bit against the eager loop's torch statement, the top-p keep set and inverse-CDF draw
against a float64 statement, the Philox stream (reproducible, chi-square against the filtered distribution), and the
model-level behaviour of ``enable_decode_graphs`` with a repetition penalty and with sampling."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

V_MODEL = 32002


def _select(logits, out_ids, step, finished, params, eos=None, pad=0, min_length=0, sample=False, seed=None, uniforms=None):
    from mm_interleaved_b200 import ops
    B = logits.shape[0]
    nxt = torch.full((B, 1), -7, dtype=torch.long, device="cuda")
    ops.decode_select(logits, out_ids, torch.tensor([step], device="cuda"), finished, nxt,
                      torch.tensor(params, dtype=torch.float32, device="cuda"),
                      eos=None if eos is None else torch.tensor(eos, device="cuda"), pad_id=pad, min_length=min_length,
                      sample=sample, seed=seed, uniforms=uniforms)
    return nxt[:, 0]


def _eager_greedy(scores, hist, finished, eos, pad, min_length, step, p):
    """The processors of InterleavedForward.generate_texts' eager loop, as written there (on the GPU, like it)."""
    if p != 1.0 and step > 0:
        prev = hist[:, :step]
        picked = scores.gather(1, prev)
        scores = scores.scatter(1, prev, torch.where(picked < 0, picked * p, picked / p))
    if step < min_length and eos:
        scores = scores.clone()
        scores[:, eos] = float("-inf")
    nxt = scores.argmax(-1)
    if eos:
        nxt = torch.where(finished, torch.full_like(nxt, pad), nxt)
        for e in eos:
            finished = finished | (nxt == e)
    return nxt, finished


def test_greedy_processors_match_the_eager_loop_bit_for_bit():
    g = torch.Generator().manual_seed(0)
    B, max_new, step, pad, p = 4, 12, 6, 0, 1.3
    logits = (torch.randn((B, V_MODEL), generator=g) * 3).cuda()
    hist = torch.randint(0, V_MODEL, (B, max_new), generator=g).cuda()
    top = logits.argmax(-1)
    neg = logits.argmin(-1)
    hist[0, :step] = torch.tensor([int(top[0]), 11, int(top[0]), int(neg[0]), 11, 5])   # duplicates, both signs
    hist[1, :step] = torch.tensor([int(neg[1]), int(neg[1]), 3, 4, 3, int(top[1])])
    logits[2, 777] = logits[2, 4321] = float(logits[2].max()) + 1.0                       # planted arg-max tie
    eos = [int(top[1]), 2]                                                                # a row's arg-max is an eos id
    fin = torch.tensor([False, False, False, True], device="cuda")                        # a finished row emits pad
    assert float(logits[0, top[0]]) > 0 and float(logits[0, neg[0]]) < 0
    for min_length, penalty in ((step + 1, p), (0, p), (0, 1.0), (step + 1, 1.7)):
        out = hist.clone()
        f = fin.clone()
        got = _select(logits, out, step, f, [penalty, 1.0, 1.0], eos=eos, pad=pad, min_length=min_length)
        want, want_f = _eager_greedy(logits, hist, fin, eos, pad, min_length, step, penalty)
        assert torch.equal(got, want), (min_length, penalty, got, want)
        assert torch.equal(f, want_f)
        ref_out = hist.clone()
        ref_out[:, step] = want
        assert torch.equal(out, ref_out)
    # the processors matter in these rows: the penalty moved row 0 off its raw arg-max, the tie went to the first index
    got = _select(logits, hist.clone(), step, fin.clone(), [p, 1.0, 1.0], eos=eos, pad=pad, min_length=step + 1)
    assert int(got[0]) != int(top[0]) and int(got[2]) == 777 and int(got[3]) == pad
    # a step outside [0, max_new) writes nothing
    out = hist.clone()
    _select(logits, out, max_new, fin.clone(), [p, 1.0, 1.0], eos=eos)
    assert torch.equal(out, hist)


def _topp_logits(B, V, seed):
    """A few hundred tokens of real mass at random positions over a negligible background (so the float64 statement's
    boundary cases stay rare)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, V), generator=g) * 0.5 - 20.0
    for b in range(B):
        idx = torch.randperm(V, generator=g)[:256]
        x[b, idx] = torch.randn(256, generator=g) * 2.5
    return x


def _ref_draw(row, temperature, top_p, u, band=1e-5):
    """HF's ascending-cumsum top-p rule and the inverse CDF over the kept set in vocabulary order, in float64.  Returns
    (id, ambiguous): ambiguous when moving the threshold by +-band changes the drawn id, or when u * Z lies within
    band * Z of a CDF step."""
    x = row.double() / temperature
    p = torch.softmax(x, 0)
    srt, idx = p.sort()
    cum = srt.cumsum(0)

    def draw(thr):
        drop = cum <= thr
        drop[-1] = False
        keep = torch.ones_like(p, dtype=torch.bool)
        keep[idx[drop]] = False
        c = torch.where(keep, p, torch.zeros_like(p)).cumsum(0)
        z = float(c[-1])
        i = int(torch.searchsorted(c, torch.tensor([u * z], dtype=torch.float64), right=True)[0])
        kept_c = c[keep]
        near = bool(((kept_c - u * z).abs() < band * z).any())
        return min(i, p.numel() - 1), near

    thr = 1.0 - top_p
    mid, near = draw(thr)
    lo, _ = draw(thr - band)
    hi, _ = draw(thr + band)
    return mid, near or lo != mid or hi != mid


def test_top_p_keep_set_and_draw_match_a_float64_statement():
    B = 4
    logits = _topp_logits(B, V_MODEL, seed=1)
    dev = logits.cuda()
    ambiguous = [0] * B
    checked = 0
    for temperature in (0.7, 1.0, 2.0):
        for top_p in (0.5, 0.9, 0.99, 1.0):
            for u in (1e-3, 0.5, 1.0 - 1e-3):
                us = torch.full((B,), u, dtype=torch.float32)
                got = _select(dev, torch.zeros((B, 4), dtype=torch.long, device="cuda"), 0,
                              torch.zeros(B, dtype=torch.bool, device="cuda"), [1.0, temperature, top_p], sample=True,
                              uniforms=us.cuda()).cpu()
                for b in range(B):
                    want, amb = _ref_draw(logits[b], temperature, top_p, float(us[b]))
                    if amb:
                        ambiguous[b] += 1
                        continue
                    checked += 1
                    assert int(got[b]) == want, (b, temperature, top_p, u, int(got[b]), want)
    assert max(ambiguous) <= 1 and checked >= 4 * 36 - 4, ambiguous


def test_philox_stream_is_reproducible_and_follows_the_filtered_distribution():
    from scipy.stats import chisquare
    B = 8
    logits = _topp_logits(B, V_MODEL, seed=2).cuda()
    seed = torch.tensor([1234567], dtype=torch.long, device="cuda")
    kw = dict(params=[1.0, 1.0, 0.9], sample=True, seed=seed)
    out = lambda: torch.zeros((B, 4), dtype=torch.long, device="cuda")
    fin = lambda: torch.zeros(B, dtype=torch.bool, device="cuda")
    a = _select(logits, out(), 0, fin(), **kw)
    b = _select(logits, out(), 0, fin(), **kw)
    c = _select(logits, out(), 1, fin(), **kw)
    assert torch.equal(a, b) and not torch.equal(a, c)

    # chi-square of 2^20 draws (4096 rows x 256 steps) on a 12-token row against the exact filtered distribution
    V, rows, steps, top_p, temperature = 12, 4096, 256, 0.85, 1.3
    row = torch.tensor([0.3, -1.0, 1.2, 0.0, 2.0, -0.5, 0.9, -2.0, 1.5, 0.1, -0.2, 0.6])
    x = row.double() / temperature
    p = torch.softmax(x, 0)
    srt, idx = p.sort()
    drop = srt.cumsum(0) <= 1.0 - top_p
    drop[-1] = False
    keep = torch.ones(V, dtype=torch.bool)
    keep[idx[drop]] = False
    assert 2 <= int(keep.sum()) < V
    want = torch.where(keep, p, torch.zeros_like(p))
    want = want / want.sum()
    lg = row.cuda().expand(rows, V).contiguous()
    out = torch.zeros((rows, steps), dtype=torch.long, device="cuda")
    fin = torch.zeros(rows, dtype=torch.bool, device="cuda")
    seed = torch.tensor([987654321], dtype=torch.long, device="cuda")
    for t in range(steps):
        _select(lg, out, t, fin, [1.0, temperature, top_p], sample=True, seed=seed)
    counts = torch.bincount(out.flatten().cpu(), minlength=V).double()
    assert float(counts[~keep].sum()) == 0
    n = float(counts.sum())
    stat, pval = chisquare(counts[keep].numpy(), (want[keep] * n).numpy())
    assert pval > 1e-3, (stat, pval)


# ---- model level ----------------------------------------------------------------------------------------------------

def _second_call_inputs(ids, vis):
    g = torch.Generator().manual_seed(123)
    vis2_d = {"vis_embed": (torch.randn(vis["vis_embed"].shape, generator=g) * 0.5).cuda(),
              "multiscale_features": [(torch.randn(f.shape, generator=g) * 2).cuda() for f in vis["multiscale_features"]]}
    mask2 = torch.ones_like(ids)
    mask2[1, :2] = 0                                                   # left padding on the second sequence
    return vis2_d, mask2.cuda()


def test_graphed_greedy_with_repetition_penalty_is_token_identical_to_eager():
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    vis2_d, mask2 = _second_call_inputs(ids, vis)
    args = (ids.cuda(), vis_d, nimg.cuda(), 2)
    args2 = (ids.cuda(), vis2_d, nimg.cuda(), 2)
    kw = dict(max_new_tokens=9, eos_token_id=[2, 17], min_length=3, repetition_penalty=1.7)
    free = dev.generate_texts(*args, max_new_tokens=9, eos_token_id=[2, 17], min_length=3).cpu()
    eager_a = dev.generate_texts(*args, **kw).cpu()
    eager_b = dev.generate_texts(*args2, attention_mask=mask2, **kw).cpu()
    eager_c = dev.generate_texts(*args, **dict(kw, repetition_penalty=1.3)).cpu()
    assert not torch.equal(eager_a, free) and not torch.equal(eager_a, eager_b)
    dev.enable_decode_graphs()
    try:
        graph_a = dev.generate_texts(*args, **kw).cpu()
        graph_b = dev.generate_texts(*args2, attention_mask=mask2, **kw).cpu()
        graph_c = dev.generate_texts(*args, **dict(kw, repetition_penalty=1.3)).cpu()
        assert len(dev._decode_graphs) == 1                            # one captured graph served all three calls
        assert torch.equal(graph_a, eager_a), (graph_a, eager_a)
        assert torch.equal(graph_b, eager_b), (graph_b, eager_b)
        assert torch.equal(graph_c, eager_c), (graph_c, eager_c)
    finally:
        dev.enable_decode_graphs(False)


def test_graphed_sampling_is_seeded_reuses_one_graph_and_reaches_the_greedy_limits():
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    args = (ids.cuda(), vis_d, nimg.cuda(), 2)
    n = 8
    greedy = dev.generate_texts(*args, max_new_tokens=n, eos_token_id=None)
    # without sampling=True, sampled calls keep the eager loop: no graph is captured
    dev.enable_decode_graphs()
    dev.generate_texts(*args, max_new_tokens=n, eos_token_id=None, use_nucleus_sampling=True,
                       generator=torch.Generator(device="cuda").manual_seed(1))
    assert len(dev._decode_graphs) == 0
    dev.enable_decode_graphs(True, sampling=True)
    try:
        samp = lambda seed, **kw: dev.generate_texts(*args, max_new_tokens=n, eos_token_id=None, use_nucleus_sampling=True,
                                                     generator=torch.Generator(device="cuda").manual_seed(seed), **kw)
        s1 = samp(5, top_p=0.95, temperature=2.0)
        s2 = samp(5, top_p=0.95, temperature=2.0)
        s3 = samp(6, top_p=0.95, temperature=2.0)
        assert torch.equal(s1, s2) and not torch.equal(s1, s3)
        assert int(s1.min()) >= 0 and int(s1.max()) < 64 and not torch.equal(s1, greedy)
        # top_p -> 0 keeps only the most likely token; temperature -> 0 concentrates all mass on it
        assert torch.equal(samp(7, top_p=1e-6), greedy)
        assert torch.equal(samp(8, top_p=1.0, temperature=1e-4), greedy)
        samp(9, top_p=0.5, temperature=0.8, repetition_penalty=1.3)
        assert len(dev._decode_graphs) == 1                            # new top_p / temperature / penalty: same graph
    finally:
        dev.enable_decode_graphs(False)


def test_vocabulary_above_the_select_limit_decodes_greedily_in_the_eager_loop_under_graphs():
    """``decode_select`` takes V <= ``ops.SELECT_MAX_V``: above it, greedy ``generate_texts`` under
    ``enable_decode_graphs()`` keeps the eager loop (no graph is captured) instead of raising."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import ops
    from mm_interleaved_b200.mm_interleaved import InterleavedForward
    from tests.golden.make_golden import LLAMA_TINY, seeded_state_dict
    V = ops.SELECT_MAX_V + 2
    cfg = m.LlamaMMFSConfig(**dict(LLAMA_TINY, vocab_size=V))
    model = InterleavedForward(cfg, special_tokens=dict(bos_token_id=1, image_token_id=V - 2, soi_token_id=V - 1),
                               orig_vocab_size=V - 2)
    model.load_state_dict(seeded_state_dict(model.state_dict(), seed=5))
    dev = model.cuda().eval()
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(3, 60, (2, 12), generator=g)
    ids[:, 0] = 1
    ids[:, 2] = V - 1                                                  # <soi> + 3 <image> tokens per sequence
    ids[:, 3:6] = V - 2
    vis = {"vis_embed": torch.randn((2, 3, cfg.hidden_size), generator=g).cuda(),
           "multiscale_features": [torch.randn((2, cfg.image_embed_dim, s, s), generator=g).cuda() for s in (8, 4, 2)]}
    args = (ids.cuda(), vis, torch.tensor([1, 1]).cuda(), 1)
    eager = dev.generate_texts(*args, max_new_tokens=4, eos_token_id=None)
    dev.enable_decode_graphs()
    try:
        graphed = dev.generate_texts(*args, max_new_tokens=4, eos_token_id=None)
        assert len(dev._decode_graphs) == 0
        assert torch.equal(graphed, eager)
    finally:
        dev.enable_decode_graphs(False)


def test_release_inference_config_takes_the_graph_through_mm_interleaved_generate():
    from tests.test_mm_interleaved_gpu import DEV, _batch, _build
    model, _ = _build()
    ids, images, nimg, mask = _batch()
    batch = dict(text_ids=ids.to(DEV), image_tensors=images.to(DEV), num_image_per_seq=nimg.to(DEV),
                 attention_mask=mask.to(DEV), meta=None)
    release = dict(num_beams=1, use_nucleus_sampling=True, repetition_penalty=1.3, min_length=8, max_length=90, top_p=0.9)
    model.enable_decode_graphs(True, sampling=True)
    try:
        g = torch.Generator(device=DEV).manual_seed(0)
        out = model.generate(mode="generate_texts", **batch, generator=g, **release)["text_ids"]
        assert len(model._decode_graphs) == 1 and next(iter(model._decode_graphs))[-1] == "sample"
        V = model.text_decoder.head.weight.shape[0]
        assert out.shape == (2, 90) and int(out.min()) >= 0 and int(out.max()) < V
        again = model.generate(mode="generate_texts", **batch, generator=torch.Generator(device=DEV).manual_seed(0),
                               **release)["text_ids"]
        assert torch.equal(out, again) and len(model._decode_graphs) == 1
    finally:
        model.enable_decode_graphs(False)
