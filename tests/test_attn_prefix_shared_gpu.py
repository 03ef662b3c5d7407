"""GPU tests of prefix-shared, segment-causal attention (``ops.attention_prefix_shared``) and of ``generate_scores``
on one context prefill (``MMInterleaved.enable_shared_context_scores``).

Kernel: both routes (the wgmma variant for 16-bit hd 64 / 128, the generic variant for fp32, odd head dims and fewer
than 16 queries) against the float64 reference of tests/attn_oracle.py given the explicit visibility matrix, within its
elementwise bound; slots no row may read are poisoned (NaN / Inf for the generic kernel, the largest finite value for
wgmma); reruns are bit-identical; and the output agrees with ``ops.attention`` over the replicated [prefix, own] cache.

Model: the tiny fp32 model's shared-context scores against the CPU oracle of test_mm_interleaved_gpu.py and the default
path; two 13B-width layers in bf16 at 100 options, no less accurate than the default path against its fp32 run; and
the option pass's peak memory below the replicated cache's size."""
import pytest
import torch

from tests import attn_oracle as ao

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _inputs(P, G, L, Tp, H, hd, dtype, seed, pmask_kind="full", own_pad=0, dead_row=False):
    """q, k, v (P, G*L, H, hd), prefix (P, Tp, H, hd), masks and the (P, Tq, Tp + Tq) visibility of [prefix, own]."""
    Tq = G * L
    g = torch.Generator().manual_seed(seed)
    q, kc, vc = (torch.randn(s, generator=g).to(dtype) for s in ((P, Tq, H, hd), (P, Tp + Tq, H, hd), (P, Tp + Tq, H, hd)))
    pm = torch.ones((P, Tp), dtype=torch.uint8)
    if pmask_kind == "padded":                     # right padding of a shorter context in the last entry
        pm[-1, max(1, Tp - Tp // 3):] = 0
    elif pmask_kind == "holed":
        pm[0, Tp // 4:Tp // 4 + max(1, Tp // 5)] = 0
    km = torch.ones((P, G, L), dtype=torch.uint8)
    if own_pad:                                    # right-padded options: every other segment loses its tail
        km[:, ::2, max(1, L - own_pad):] = 0
    if dead_row:                                   # entry 0, segment 0, position 0 sees nothing
        pm[0] = 0
        km[0, 0, 0] = 0
    km = km.view(P, Tq)
    i = torch.arange(Tq)
    own_vis = (i[None, :] // L == i[:, None] // L) & (i[None, :] <= i[:, None])               # (Tq, Tq)
    vis = torch.cat((pm.bool()[:, None, :].expand(P, Tq, Tp), own_vis[None] & km.bool()[:, None, :]), dim=2)
    return q, kc, vc, pm, km, vis


def _run(q, kc, vc, pm, km, vis, Tp, L, finite):
    """The op on views of one poisoned [prefix, own] buffer; returns (out, the op's positional arguments)."""
    import mm_interleaved_b200 as m
    kp, vp = ao.poison(kc, vc, ao.hidden_slots(vis), finite=finite)
    kp, vp = kp.to(DEV), vp.to(DEV)
    args = (q.to(DEV), kp[:, :Tp], vp[:, :Tp], kp[:, Tp:], vp[:, Tp:], L)
    return m.ops.attention_prefix_shared(*args, prefix_mask=pm.to(DEV), key_mask=km.to(DEV)), args


def _arith_wgmma(Tp, L, dtype, hd):
    tiles = -(-Tp // ao.TILE) + -(-(ao.TILE * 2 + L) // ao.TILE) + 1       # prefix tiles + the most own tiles an item scans
    return ao.arith_wgmma(tiles * ao.TILE, dtype, hd)


WGMMA_CASES = [  # P, G, L, Tp, H, prefix mask, own padding, dead row
    (1, 1, 16, 1, 2, "full", 0, False),
    (3, 5, 15, 63, 2, "padded", 4, False),
    (1, 5, 64, 64, 2, "holed", 0, True),
    (3, 5, 65, 65, 2, "padded", 9, False),
    (1, 3, 130, 300, 2, "holed", 30, True),
    (3, 100, 2, 300, 2, "padded", 1, False),
    (1, 100, 16, 200, 40, "padded", 7, True),     # 13 query tiles x 40 heads: persistent
    (3, 100, 15, 63, 4, "holed", 5, False),
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("case", WGMMA_CASES)
def test_wgmma_route_against_float64(dtype, hd, case):
    import mm_interleaved_b200 as m
    P, G, L, Tp, H, kind, own_pad, dead = case
    q, kc, vc, pm, km, vis = _inputs(P, G, L, Tp, H, hd, dtype, seed=sum(x for x in case if isinstance(x, int)), pmask_kind=kind, own_pad=own_pad,
                                     dead_row=dead)
    ref = ao.reference(q.to(DEV), kc.to(DEV), vc.to(DEV), vis=vis.to(DEV))
    out, args = _run(q, kc, vc, pm, km, vis, Tp, L, finite=True)
    ao.check(out, ref, _arith_wgmma(Tp, L, dtype, hd), f"wgmma {case} {dtype} hd {hd}")
    again = m.ops.attention_prefix_shared(*args, prefix_mask=pm.to(DEV), key_mask=km.to(DEV))
    assert torch.equal(out, again), "reruns must be bit-identical"
    # the same rows through ops.attention over the replicated (P*G, Tp + L) [prefix, own segment] cache, past = Tp
    kq, vq = args[1], args[2]
    kr = torch.cat((kq.repeat_interleave(G, 0), args[3].reshape(P * G, L, H, hd)), 1)
    vr = torch.cat((vq.repeat_interleave(G, 0), args[4].reshape(P * G, L, H, hd)), 1)
    mr = torch.cat((pm.repeat_interleave(G, 0), km.view(P * G, L)), 1).to(DEV)
    rep = m.ops.attention(args[0].reshape(P * G, L, H, hd), kr, vr, key_mask=mr, causal=True, past=Tp)
    b = ao.bound(ref, _arith_wgmma(Tp, L, dtype, hd))
    diff = (out.view(P, G * L, H, hd).double() - rep.view(P, G * L, H, hd).double()).abs()
    assert bool((diff <= 2 * b).all()), float((diff / b).max())


GENERIC_CASES = [  # dtype, hd, P, G, L, Tp, prefix mask, own padding, dead row
    (torch.float32, 128, 1, 1, 1, 1, "full", 0, False),
    (torch.float32, 128, 3, 5, 2, 63, "padded", 1, True),
    (torch.float32, 64, 1, 100, 15, 300, "holed", 4, False),
    (torch.float32, 96, 3, 5, 65, 64, "padded", 9, True),
    (torch.bfloat16, 96, 1, 5, 130, 65, "holed", 20, False),
    (torch.float16, 32, 3, 100, 2, 300, "padded", 1, True),
    (torch.bfloat16, 128, 3, 5, 1, 300, "padded", 0, False),     # 5 queries: below the wgmma route's 16
    (torch.float16, 64, 1, 3, 5, 64, "holed", 2, True),
]


@pytest.mark.parametrize("case", GENERIC_CASES)
def test_generic_route_against_float64(case):
    import mm_interleaved_b200 as m
    dtype, hd, P, G, L, Tp, kind, own_pad, dead = case
    H = 2
    q, kc, vc, pm, km, vis = _inputs(P, G, L, Tp, H, hd, dtype, seed=sum(x for x in case if isinstance(x, int)), pmask_kind=kind, own_pad=own_pad,
                                     dead_row=dead)
    ref = ao.reference(q.to(DEV), kc.to(DEV), vc.to(DEV), vis=vis.to(DEV))
    out, args = _run(q, kc, vc, pm, km, vis, Tp, L, finite=False)
    ao.check(out, ref, ao.arith_generic(Tp + L, dtype, hd), f"generic {case}")
    again = m.ops.attention_prefix_shared(*args, prefix_mask=pm.to(DEV), key_mask=km.to(DEV))
    assert torch.equal(out, again), "reruns must be bit-identical"


def test_each_route_runs_its_kernel():
    import mm_interleaved_b200 as m
    from torch.profiler import ProfilerActivity, profile
    names = {}
    for dtype, hd, G, L in ((torch.bfloat16, 128, 4, 16), (torch.float32, 128, 4, 16), (torch.bfloat16, 128, 3, 5)):
        q, kc, vc, pm, km, vis = _inputs(1, G, L, 70, 2, hd, dtype, seed=1)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _run(q, kc, vc, pm, km, vis, 70, L, finite=dtype != torch.float32)
            torch.cuda.synchronize()
        names[(dtype, G * L)] = [e.name for e in prof.events() if "attn" in e.name]
    assert any("attn_fwd_kernel" in n for n in names[(torch.bfloat16, 64)]), names
    assert any("attn_generic_kernel" in n for n in names[(torch.float32, 64)]), names
    assert any("attn_generic_kernel" in n for n in names[(torch.bfloat16, 15)]), names


# ---- the model ------------------------------------------------------------------------------------------------------

def _contexts(lens, n_tok, st, seed):
    g = torch.Generator().manual_seed(seed)
    ctx = []
    for L in lens:
        t = torch.randint(3, 60, (L,), generator=g)
        t[0] = st["bos_token_id"]
        t[2] = st["soi_token_id"]
        t[3:3 + n_tok] = st["image_token_id"]
        ctx.append(t)
    return ctx


def _scores(model, ctx, images, opts, masks, shared):
    model.enable_shared_context_scores(shared)
    out = model.generate(mode="generate_scores", text_ids=[t.to(DEV) for t in ctx], image_tensors=images.to(DEV),
                         num_image_per_seq=torch.ones((len(ctx), 1), dtype=torch.long, device=DEV),
                         attention_mask=[torch.ones_like(t).to(DEV) for t in ctx],
                         options_ids=[o.to(DEV) for o in opts], options_attn_masks=[mk.to(DEV) for mk in masks])
    model.enable_shared_context_scores(False)
    return out["scores"].float().cpu()


@pytest.mark.parametrize("shape", ["padded", "single_token", "one_option_of_two"])
def test_tiny_model_scores_match_the_oracle_and_the_default_path(shape):
    from oracle.glue import text_head_ref
    from tests.test_mm_interleaved_gpu import N_TOK, ST, _build, _oracle_hidden
    model, sd = _build()
    g = torch.Generator().manual_seed(7)
    ctx = _contexts((9, 14), N_TOK, ST, seed=5)
    images = torch.rand((2, 3, 56, 56), generator=g)
    G, L = {"padded": (5, 4), "single_token": (6, 1), "one_option_of_two": (1, 2)}[shape]
    opts = [torch.randint(3, 60, (G, L), generator=g) for _ in ctx]
    masks = [torch.ones((G, L), dtype=torch.long) for _ in ctx]
    if shape == "padded":
        masks[0][1, 2:] = 0
        masks[1][3, 1:] = 0
    got = _scores(model, ctx, images, opts, masks, shared=True)
    default = _scores(model, ctx, images, opts, masks, shared=False)
    assert got.shape == (2, 1, G)
    assert bool(((got - default).abs() <= 1e-4 * default.abs() + 1e-6).all()), (got, default)
    for i in range(2):
        full = torch.cat([ctx[i][None].expand(G, -1), opts[i]], 1)
        hid = _oracle_hidden(model, sd, full, images[[i]].expand(G, -1, -1, -1), torch.ones(G, dtype=torch.long))(full)
        logits = text_head_ref(sd, hid, 62)[:, len(ctx[i]) - 1:-1]
        logp = torch.log_softmax(logits, -1).gather(-1, opts[i][..., None]).squeeze(-1)
        want = (logp * masks[i]).sum(-1)
        assert bool(((got[i, 0] - want).abs() <= 1e-3 * want.abs() + 1e-3).all()), (got[i, 0], want)
    # neither FP8 switch changes the shared-context scores
    model.enable_fp8_decode(True).enable_fp8_kv_cache(True)
    try:
        fp8 = _scores(model, ctx, images, opts, masks, shared=True)
    finally:
        model.enable_fp8_decode(False).enable_fp8_kv_cache(False)
    assert torch.equal(fp8, got)


def _wide_model(dtype):
    """Two Llama-MMFS layers at the 13B widths (hidden 5120, 40 heads, MLP 13824; MMFS in layer 0) with the tiny visual
    tokenizer of test_mm_interleaved_gpu.py, seeded weights."""
    import mm_interleaved_b200 as m
    from tests.golden.make_golden import LLAMA_TINY, seeded_state_dict
    from tests.test_mm_interleaved_gpu import N_TOK, ST
    torch.manual_seed(0)
    vt_cfg = dict(clip_config=m.visual_tokenizer.CLIPVisionConfigLite(hidden_size=512, intermediate_size=512, num_hidden_layers=4,
                                                                     num_attention_heads=4, image_size=56, patch_size=14),
                  perceiver_config=dict(num_queries=N_TOK, hidden_size=192, encoder_hidden_size=512, cross_attention_frequency=2,
                                        num_hidden_layers=2, num_attention_heads=3, intermediate_size=384,
                                        qk_normalization=True), grid_size=4)
    llm = dict(vocab_size=62, hidden_size=5120, intermediate_size=13824, num_hidden_layers=2, num_attention_heads=40,
               max_position_embeddings=2048, rms_norm_eps=1e-6, pad_token_id=0)
    model = m.MMInterleaved(llm_config=llm, txt_vocab_size=64, seq_len=32, special_token_dict=ST, visual_tokenizer_config=vt_cfg,
                            image_embed_dim=LLAMA_TINY["image_embed_dim"], cross_attention_frequency=2,
                            spatial_shapes=LLAMA_TINY["spatial_shapes"])
    sd = model.state_dict()
    sd.update(seeded_state_dict({k: v for k, v in sd.items() if k.split(".")[0] in ("mm_decoder", "text_decoder", "soi_token")},
                                seed=99))
    model.load_state_dict(sd)
    return model.to(DEV, dtype).eval()


def test_13b_width_layers_bf16_no_less_accurate_than_the_default_path():
    from tests.test_mm_interleaved_gpu import N_TOK, ST
    model = _wide_model(torch.float32)
    g = torch.Generator().manual_seed(3)
    ctx = _contexts((60, 75), N_TOK, ST, seed=8)
    images = torch.rand((2, 3, 56, 56), generator=g)
    G, L = 100, 16
    opts = [torch.randint(3, 60, (G, L), generator=g) for _ in ctx]
    masks = []
    for _ in ctx:
        n = torch.randint(2, L + 1, (G,), generator=g)
        masks.append((torch.arange(L)[None, :] < n[:, None]).long())
    ref = _scores(model, ctx, images, opts, masks, shared=False).double()            # the default path in fp32
    model = model.to(torch.bfloat16)
    off = _scores(model, ctx, images, opts, masks, shared=False).double()
    on = _scores(model, ctx, images, opts, masks, shared=True).double()
    err_off, err_on = float((off - ref).abs().max()), float((on - ref).abs().max())
    floor = 0.05                              # nats: a few bf16 ulps of a score of ~-60 summed over 16 tokens
    print(f"13B-width bf16 max |score - fp32 default|: default path {err_off:.4f}, shared context {err_on:.4f}")
    assert err_on <= 1.5 * err_off + floor, (err_on, err_off)
    assert bool(torch.isfinite(on).all())


def test_option_pass_peak_memory_below_the_replicated_cache():
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.llama_mmfs import LlamaModel, PrefixKV
    cfg = m.LlamaMMFSConfig(vocab_size=64, hidden_size=5120, intermediate_size=13824, num_hidden_layers=2,
                            num_attention_heads=40, cross_attention_frequency=8)
    torch.manual_seed(0)
    with torch.device(DEV):
        dec = LlamaModel(cfg).to(torch.bfloat16).eval()
    with torch.no_grad():
        for p in dec.parameters():
            p.normal_(0.0, 0.02)
    Tp, G, L = 200, 100, 16
    with torch.no_grad():
        cache = dec.static_cache(1, Tp)
        dec(input_ids=torch.randint(3, 60, (1, Tp), device=DEV), past_key_values=cache, use_cache=True)
        pre = [PrefixKV(c.k, c.v, torch.ones((1, Tp), dtype=torch.uint8, device=DEV), L - 1) for c in cache]
        x = torch.randint(3, 60, (1, G * (L - 1)), device=DEV)
        pos = (Tp + torch.arange(L - 1, device=DEV)).repeat(G)[None]
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = dec(input_ids=x, past_key_values=pre, position_ids=pos, use_cache=False).last_hidden_state
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    replicated = 2 * cfg.num_hidden_layers * G * (Tp + L) * cfg.hidden_size * 2       # bytes of a per-option bf16 copy
    assert bool(torch.isfinite(out.float()).all())
    assert peak < replicated, (peak, replicated)
