"""GPU tests of the graphed beam search's shared-prefix KV cache: ``ops.attention_decode_shared`` (csrc/
attn_generic_sm100.cu) bit-identical to ``ops.attention``'s decode over the equivalent replicated cache, one captured
graph serving two prompt lengths of its bucket, ``generation.BeamDecoder`` over the new layout against the eager beam
loop (beam search and beam sample) and in an interleaved session, and the decoder's memory at the 13B widths."""
import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_NEW = 5


def _bucket(L, max_new=MAX_NEW):
    """T_p of the graphed decoders' cache bucket for an L-token prompt (generation._graphed_decoder)."""
    return ((L + max_new + 255) // 256) * 256 - max_new


def _case(dtype, hd, G, plen, step, P=2, H=3, seed=0):
    """Prefix, gen, q and key mask of P prompts x G rows; prompt 1 left-padded (by 300 positions when it can, so that
    a whole 256-key split is masked), ``step`` generated positions visible, everything after them masked."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    R, Tp = P * G, _bucket(plen)
    rnd = lambda *s: torch.randn(s, generator=g, device="cuda").to(dtype)
    kp, vp = rnd(P, Tp, H, hd), rnd(P, Tp, H, hd)
    kg, vg = rnd(R, MAX_NEW, H, hd), rnd(R, MAX_NEW, H, hd)
    q = rnd(R, 1, 3, H, hd)[:, :, 0]                                 # a view with the QKV GEMM's row stride
    mask = torch.zeros((R, Tp + MAX_NEW), dtype=torch.uint8, device="cuda")
    mask[:, :plen] = 1
    mask[G:2 * G, :min(plen - 1, 300)] = 0
    mask[:, plen:plen + step] = 1
    return q, kp, vp, kg, vg, mask


def _replicated(kp, vp, kg, vg, plen, G):
    """The (R, T_p + max_new, H, hd) cache the shared layout stands for; masked positions hold zeros."""
    R, max_new = kg.shape[:2]
    Tp = kp.shape[1]
    out = []
    for pre, gen in ((kp, kg), (vp, vg)):
        full = torch.zeros((R, Tp + max_new) + tuple(pre.shape[2:]), dtype=pre.dtype, device=pre.device)
        full[:, :plen] = pre[:, :plen].repeat_interleave(G, 0)
        full[:, plen:plen + max_new] = gen
        out.append(full)
    return out


def _same(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8)) if a.element_size() == 2 else torch.equal(a, b)


@pytest.mark.parametrize("G", [1, 3, 5, 10])
@pytest.mark.parametrize("hd", [128, 64])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_shared_decode_is_bit_identical_to_the_replicated_cache(dtype, hd, G):
    from mm_interleaved_b200 import ops
    for plen in (1, 63, 64, 65, 255, 256, 257, 2048):
        for step in (0, 1, MAX_NEW):
            q, kp, vp, kg, vg, mask = _case(dtype, hd, G, plen, step, seed=plen * 7 + step)
            kr, vr = _replicated(kp, vp, kg, vg, plen, G)
            t_max = kr.shape[1]
            plen_d = torch.tensor([plen], device="cuda")
            for past in (t_max - 1, plen + step - 1, max(plen // 2 - 1, 0)):     # graph, the query's own, a smaller one
                want = ops.attention(q, kr, vr, key_mask=mask, causal=True, past=past)
                got = ops.attention_decode_shared(q, kp, vp, kg, vg, plen_d, key_mask=mask, past=past)
                assert _same(got, want), (dtype, hd, G, plen, step, past, (got.float() - want.float()).abs().max())


def test_shared_decode_counts_its_launches_as_attention_does():
    from mm_interleaved_b200 import ops
    q, kp, vp, kg, vg, mask = _case(torch.bfloat16, 128, 5, 100, 1)
    kr, vr = _replicated(kp, vp, kg, vg, 100, 5)
    n0 = ops.launch_counter[0]
    ops.attention(q, kr, vr, key_mask=mask, past=kr.shape[1] - 1)
    n1 = ops.launch_counter[0]
    ops.attention_decode_shared(q, kp, vp, kg, vg, torch.tensor([100], device="cuda"), key_mask=mask, past=kr.shape[1] - 1)
    assert ops.launch_counter[0] - n1 == n1 - n0 == 2


@pytest.mark.parametrize("dtype, hd", [(torch.bfloat16, 128), (torch.float32, 64)])
def test_one_captured_graph_serves_two_prompt_lengths_of_its_bucket(dtype, hd):
    from mm_interleaved_b200 import ops
    G, lens = 5, (300, 490)                                           # both in the 512-position bucket
    assert _bucket(lens[0]) == _bucket(lens[1])
    q, kp, vp, kg, vg, _ = _case(dtype, hd, G, lens[1], MAX_NEW)
    mask = torch.zeros((kg.shape[0], kp.shape[1] + MAX_NEW), dtype=torch.uint8, device="cuda")
    plen_d = torch.zeros((1,), dtype=torch.long, device="cuda")
    past = mask.shape[1] - 1
    ops.attention_decode_shared(q, kp, vp, kg, vg, plen_d, key_mask=mask, past=past)    # warm-up off the graph
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.attention_decode_shared(q, kp, vp, kg, vg, plen_d, key_mask=mask, past=past)
    for plen in lens:
        mask.zero_()
        mask[:, :plen] = 1
        mask[:, plen:plen + 2] = 1
        plen_d.fill_(plen)
        graph.replay()
        kr, vr = _replicated(kp, vp, kg, vg, plen, G)
        want = ops.attention(q, kr, vr, key_mask=mask, causal=True, past=past)
        assert _same(out, want), plen


# ---- the decoder ---------------------------------------------------------------------------------------------------

def _check_layout(dev, B, nb, expand, L, max_new):
    """The graphed beam decoder keeps the prompt once per prompt and only the generated positions per row."""
    from mm_interleaved_b200.generation import BeamDecoder
    from mm_interleaved_b200.llama_mmfs import SharedPrefixKV
    dec = next(d for d in dev._decode_graphs.values() if isinstance(d, BeamDecoder))
    cfg = dev.mm_decoder.config
    H, n = cfg.num_attention_heads, 2 * cfg.num_hidden_layers
    R, hd = B * expand * nb, cfg.hidden_size // cfg.num_attention_heads
    t_max = ((L + max_new + 255) // 256) * 256
    assert tuple(dec.prefix.shape) == (n, B, t_max - max_new, H, hd)
    assert tuple(dec.gen.shape) == (n, R, max_new, H, hd)
    assert all(isinstance(c, SharedPrefixKV) and c.G == expand * nb for c in dec.past)
    for name, t in vars(dec).items():                                 # no R-row copy of the prompt anywhere
        if isinstance(t, torch.Tensor) and t.dim() >= 3 and t.shape[0] == R:
            assert t.shape[1] < L, (name, tuple(t.shape))
    assert not hasattr(dec, "kv")
    return dec


@pytest.mark.parametrize("nb", [3, 5])
def test_graphed_beam_search_over_the_shared_prefix_equals_the_eager_loop(nb):
    from tests.test_beam_select_gpu import _second_call
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    vis2_d, mask2 = _second_call(ids, vis)
    args, args2 = (ids.cuda(), vis_d, nimg.cuda(), 2), (ids.cuda(), vis2_d, nimg.cuda(), 2)
    free = dev.generate_texts(*args, max_new_tokens=8, eos_token_id=None).cpu()
    kw = dict(max_new_tokens=8, eos_token_id=[int(free[0, 3]), int(free[1, 2])], min_length=2, num_beams=nb,
              length_penalty=1.3, num_return_sequences=2, pad_token_id=0)
    calls = [(args, {}), (args2, dict(attention_mask=mask2))]
    eager = [dev.generate_texts(*a, **dict(kw, **extra)).cpu() for a, extra in calls]
    dev.enable_decode_graphs()
    try:
        graphed = [dev.generate_texts(*a, **dict(kw, **extra)).cpu() for a, extra in calls]
        _check_layout(dev, 2, nb, 1, ids.shape[1], 8)
        for e, g in zip(eager, graphed):
            assert torch.equal(e, g), (e, g)
    finally:
        dev.enable_decode_graphs(False)


def test_graphed_beam_sample_over_the_shared_prefix_equals_the_eager_loop():
    """top_p far below every row's top probability keeps exactly two tokens per row (4.31's min_tokens_to_keep), so
    both loops draw every one of a sequence's 2 * num_beams candidates and the ids do not depend on the draws."""
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    args = (ids.cuda(), vis_d, nimg.cuda(), 2)
    kw = dict(max_new_tokens=8, eos_token_id=[7, 11], min_length=2, num_beams=3, length_penalty=1.3,
              num_return_sequences=2, use_nucleus_sampling=True, temperature=1.0, top_p=1e-6)
    gen = lambda: dev.generate_texts(*args, generator=torch.Generator(device="cuda").manual_seed(5), **kw).cpu()
    eager = gen()
    dev.enable_decode_graphs(True, sampling=True)
    try:
        graphed = gen()
        _check_layout(dev, 2, 3, 2, ids.shape[1], 8)
        assert graphed.shape[0] == 4 and torch.equal(eager, graphed), (eager, graphed)
    finally:
        dev.enable_decode_graphs(False)


def test_interleaved_session_beam_turn_equals_the_call_without_a_session():
    """The session's graphed beam turn prefills after its cached prefix and copies the prompt's one row into the shared
    prefix; the same call through ``generate`` prefills straight into it."""
    from tests.test_interleaved_gpu import GEN, build, sample
    model = build()
    model.enable_decode_graphs()
    inputs = sample()
    gen = dict(GEN, num_beams=5, max_length=5)
    kw = {k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors", "num_image_per_seq")}
    out = model.generate_interleaved(**kw, num_iter=1, **gen)
    alone = model.generate(mode="generate_texts", **{k: v.clone() for k, v in inputs.items()}, **gen)["text_ids"]
    assert out["turns"][0]["mode"] == "generate_texts"
    assert torch.equal(out["turns"][0]["text_ids"].cpu(), alone.cpu()), (out["turns"][0]["text_ids"], alone)
    _check_layout(model, 1, 5, 1, inputs["text_ids"].shape[1], 5)


def test_peak_memory_at_13b_widths_stays_below_the_replicated_cache():
    """4 layers of 40 x 128 heads, B = 4, 5 beams, a 2048-token prompt: the old layout's beam cache alone, computed from
    the shapes, is more than the whole call now allocates on top of the model (its weights and the fused weight copies
    a first call builds)."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.mm_interleaved import InterleavedForward
    torch.manual_seed(0)
    cfg = m.LlamaMMFSConfig(num_hidden_layers=4, vocab_size=32002)
    with torch.device("cuda"):                                         # default init, on the device
        model = InterleavedForward(cfg, special_tokens=dict(bos_token_id=1, image_token_id=32000, soi_token_id=32001),
                                   orig_vocab_size=32000).to(torch.bfloat16).eval()
    B, L, nb, max_new, n_tok = 4, 2048, 5, 20, 64
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, 31999, (B, L), generator=g)
    ids[:, 0] = 1
    for i in range(4):                                                 # four images per prompt
        ids[:, 10 + 300 * i] = 32001
        ids[:, 11 + 300 * i:11 + 300 * i + n_tok] = 32000
    nimg = torch.full((B,), 4, dtype=torch.long)
    vis = {"vis_embed": torch.randn((4 * B, n_tok, cfg.hidden_size), generator=g).to(torch.bfloat16).cuda() * 0.1,
           "multiscale_features": [torch.randn((4 * B, cfg.image_embed_dim, s, s), generator=g).to(torch.bfloat16).cuda()
                                   for s in cfg.spatial_shapes]}
    t_max = ((L + max_new + 255) // 256) * 256
    hd = cfg.hidden_size // cfg.num_attention_heads
    old_cache = 2 * cfg.num_hidden_layers * B * nb * t_max * cfg.num_attention_heads * hd * 2
    with torch.no_grad():                                              # builds the fused QKV / gate-up weights
        vis1 = {"vis_embed": vis["vis_embed"][:4], "multiscale_features": [f[:4] for f in vis["multiscale_features"]]}
        model.generate_texts(ids[:1].cuda(), vis1, nimg[:1].cuda(), 4, max_new_tokens=1)
    model.enable_decode_graphs()
    try:
        with torch.no_grad():
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = model.generate_texts(ids.cuda(), vis, nimg.cuda(), 4, max_new_tokens=max_new, eos_token_id=[2],
                                       min_length=8, num_beams=nb)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
        assert out.shape[0] == B
        _check_layout(model, B, nb, 1, L, max_new)
        assert peak < old_cache, (peak / 2**30, old_cache / 2**30)
    finally:
        model.enable_decode_graphs(False)
