"""GPU tests of the FP8 KV cache: the append kernel bit for bit against ``ops.quantize_kv_fp8``, FP8 decode attention
against float64 attention over ``x8 * scale``, the shared-prefix kernel bit for bit against the replicated cache, and
the model switch (``enable_fp8_kv_cache``) against the 16-bit model whose keys and values are replaced by
``x8 * scale`` on entering the cache, eagerly, graphed and in an interleaved session."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16, F16 = torch.bfloat16, torch.float16


def _bytes(t):
    return t.view(torch.uint8)


# ---- the append kernel -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [BF16, F16, torch.float32])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("device_slot", [False, True])
def test_append_is_bit_identical_to_the_torch_reference(dtype, hd, device_slot):
    from mm_interleaved_b200 import ops
    from mm_interleaved_b200.llama_mmfs import rotary_tables
    B, T, H, T_max, slot = 2, 5, 3, 16, 7
    g = torch.Generator(device="cuda").manual_seed(hd + T)
    qkv = (torch.randn((B, T, 3, H, hd), generator=g, device="cuda") *
           torch.logspace(-3, 2, H, device="cuda")[:, None]).to(dtype)
    qkv[0, 1, 1, 2] = 0                                                     # an all-zero key
    qkv[1, 3, 2, 0] = 0                                                     # an all-zero value
    cos, sin = rotary_tables(hd, 64, device="cuda")
    pos = torch.arange(3, 3 + T, device="cuda").repeat(B, 1)
    ref = qkv.clone()
    ops.rope_qk_(ref[:, :, 0], ref[:, :, 1], cos, sin, pos)                # rotated q and k, 16-bit
    k8_ref, ks_ref = ops.quantize_kv_fp8(ref[:, :, 1])
    v8_ref, vs_ref = ops.quantize_kv_fp8(ref[:, :, 2])
    q16 = qkv.clone()
    kc16, vc16 = (torch.zeros((B, T_max, H, hd), dtype=dtype, device="cuda") for _ in range(2))
    ops.rope_qk_append_(q16[:, :, 0], q16[:, :, 1], q16[:, :, 2], cos, sin, pos, kc16, vc16, slot)

    Hs = ops.kv_scale_heads(H)
    k8, v8 = (torch.zeros((B, T_max, H, hd), dtype=torch.float8_e4m3fn, device="cuda") for _ in range(2))
    ks, vs = (torch.full((B, T_max, Hs), 7.0, device="cuda") for _ in range(2))
    got = qkv.clone()
    s = torch.tensor([slot], device="cuda") if device_slot else slot
    ops.rope_qk_append_fp8_(got[:, :, 0], got[:, :, 1], got[:, :, 2], cos, sin, pos, k8, v8, ks, vs, s)
    assert torch.equal(got[:, :, 0], q16[:, :, 0]), "q is rotated as rope_qk_append_ rotates it"
    assert torch.equal(_bytes(k8[:, slot:slot + T]), _bytes(k8_ref)) and torch.equal(ks[:, slot:slot + T, :H], ks_ref)
    assert torch.equal(_bytes(v8[:, slot:slot + T]), _bytes(v8_ref)) and torch.equal(vs[:, slot:slot + T, :H], vs_ref)
    assert not bool(_bytes(k8[:, :slot]).any()) and bool((ks[:, :slot] == 7).all()), "other positions untouched"
    assert bool((ks[:, slot:slot + T, H:] == 7).all()), "the padding heads of a scale row are untouched"
    assert torch.equal(got[:, :, 1], (k8_ref.float() * ks_ref[..., None]).to(dtype)), "k rewritten with x8 * scale"
    assert torch.equal(got[:, :, 2], (v8_ref.float() * vs_ref[..., None]).to(dtype)), "v rewritten with x8 * scale"
    assert float(ks_ref[0, 1, 2]) == 1.0 and not bool(k8_ref[0, 1, 2].float().any()), "a zero vector: scale 1, zeros"


# ---- decode attention ------------------------------------------------------------------------------------------------
def _cache(B, Tkv, H, hd, dtype, seed):
    from mm_interleaved_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn((B, 1, H, hd), generator=g, device="cuda").to(dtype)
    k = torch.randn((B, Tkv, H, hd), generator=g, device="cuda") * 2.0
    v = torch.randn((B, Tkv, H, hd), generator=g, device="cuda") * torch.logspace(-2, 1, H, device="cuda")[:, None]
    k8, ks = ops.quantize_kv_fp8(k.to(dtype))
    v8, vs = ops.quantize_kv_fp8(v.to(dtype))
    pad = ops.kv_scale_heads(H) - H
    ks, vs = (torch.nn.functional.pad(s, (0, pad), value=float("nan")) for s in (ks, vs))   # padding heads never read
    return q, k8, v8, ks, vs


def _ref(q, k8, v8, ks, vs, mask, past):
    """float64 softmax attention over keys / values x8 * scale; (B, 1, H*hd)."""
    B, _, H, hd = q.shape
    kd = k8.double() * ks[..., :H, None].double()
    vd = v8.double() * vs[..., :H, None].double()
    sc = torch.einsum("bhd,bthd->bht", q[:, 0].double(), kd) * hd ** -0.5
    Tkv = k8.shape[1]
    vis = torch.arange(Tkv, device=q.device)[None, :] <= past
    if mask is not None:
        vis = vis & mask.bool()
    sc = sc.masked_fill(~vis[:, None, :], float("-inf"))
    p = torch.softmax(sc, -1).nan_to_num(0.0)
    return torch.einsum("bht,bthd->bhd", p, vd).reshape(B, 1, H * hd), torch.einsum("bht,bthd->bhd", p, vd.abs())


def _poison(k8, v8, ks, vs, mask, past):
    """NaN bytes and scales in every slot the row may not see: they must never reach the sums."""
    vis = (torch.arange(k8.shape[1], device=k8.device)[None, :] <= past).expand(k8.shape[0], -1)
    if mask is not None:
        vis = vis & mask.bool()
    hidden = ~vis
    for t in (k8, v8):
        _bytes(t)[hidden] = 0x7F                                            # e4m3fn NaN
    for s in (ks, vs):
        s[hidden] = float("nan")


def _check(out, ref, mag, dtype):
    u = {BF16: 2.0 ** -8, F16: 2.0 ** -11}.get(dtype, 2.0 ** -20)
    err = (out.double() - ref).abs()
    tol = u * ref.abs() + 1e-5 * mag.reshape(ref.shape) + 1e-6
    assert not bool((err > tol).any()), f"{int((err > tol).sum())} outside, worst {float((err - tol).max())}"


CASES = [(2, 37, 2, 64), (2, 300, 2, 128), (3, 700, 2, 64), (2, 2304, 40, 128)]


@pytest.mark.parametrize("dtype", [BF16, F16, torch.float32])
@pytest.mark.parametrize("B, Tkv, H, hd", CASES)
def test_decode_fp8_against_float64(B, Tkv, H, hd, dtype):
    from mm_interleaved_b200 import ops
    q, k8, v8, ks, vs = _cache(B, Tkv, H, hd, dtype, seed=Tkv + hd)
    g = torch.Generator(device="cuda").manual_seed(1)
    mask = (torch.rand((B, Tkv), generator=g, device="cuda") > 0.2).to(torch.uint8)
    mask[:, :3] = 0                                                         # left padding
    mask[-1] = 0                                                            # a fully masked row
    for past in (Tkv - 1, Tkv // 2):
        for m in (None, mask):
            kk, vv, kss, vss = k8.clone(), v8.clone(), ks.clone(), vs.clone()
            _poison(kk, vv, kss, vss, m, past)
            out = ops.attention_decode_fp8(q, kk, vv, kss, vss, key_mask=m, past=past)
            ref, mag = _ref(q, k8, v8, ks, vs, m, past)
            assert not bool(out.isnan().any())
            _check(out, ref, mag, dtype)
            if m is not None:
                assert not bool(out[-1].any()), "a fully masked row gives zeros"
            assert torch.equal(out, ops.attention_decode_fp8(q, kk, vv, kss, vss, key_mask=m, past=past)), "rerun"


def test_decode_fp8_graph_replay_equals_eager():
    from mm_interleaved_b200 import ops
    q, k8, v8, ks, vs = _cache(2, 2304, 40, 128, BF16, seed=5)
    mask = torch.ones((2, 2304), dtype=torch.uint8, device="cuda")
    want = ops.attention_decode_fp8(q, k8, v8, ks, vs, key_mask=mask, past=2303)
    out = torch.empty_like(want)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out.copy_(ops.attention_decode_fp8(q, k8, v8, ks, vs, key_mask=mask, past=2303))
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out.copy_(ops.attention_decode_fp8(q, k8, v8, ks, vs, key_mask=mask, past=2303))
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    mask[:, 1000:] = 0                                                      # the graph reads the mask on the device
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ops.attention_decode_fp8(q, k8, v8, ks, vs, key_mask=mask, past=2303))


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("G", [1, 5])
def test_shared_fp8_is_bit_identical_to_the_replicated_cache(dtype, hd, G):
    from mm_interleaved_b200 import ops
    P, H, Tp, max_new = 2, 3, 520, 8
    R = P * G
    _, kp, vp, ksp, vsp = _cache(P, Tp, H, hd, dtype, seed=hd + G)
    q, kg, vg, ksg, vsg = _cache(R, max_new, H, hd, dtype, seed=hd + G + 1)
    for plen, step in ((Tp, 3), (300, 8), (1, 1)):
        Tkv = Tp + max_new
        mask = torch.zeros((R, Tkv), dtype=torch.uint8, device="cuda")
        mask[:, :plen] = 1
        mask[:, plen:plen + step] = 1
        mask[0, :2] = 0
        rows = torch.arange(R, device="cuda") // G
        rep = []
        for pre, gen in ((kp, kg), (vp, vg), (ksp, ksg), (vsp, vsg)):
            r = torch.zeros((R, Tkv) + tuple(pre.shape[2:]), dtype=pre.dtype, device="cuda")
            _bytes(r)[:, :plen] = _bytes(pre)[rows, :plen]
            _bytes(r)[:, plen:plen + max_new] = _bytes(gen)
            rep.append(r)
        past = plen + step - 1
        want = ops.attention_decode_fp8(q, *rep, key_mask=mask, past=past)
        got = ops.attention_decode_shared_fp8(q, kp, vp, ksp, vsp, kg, vg, ksg, vsg,
                                              torch.tensor([plen], device="cuda"), key_mask=mask, past=past)
        assert torch.equal(got, want), (plen, step)


# ---- the model -------------------------------------------------------------------------------------------------------
def _quantise_on_entry(monkeypatch):
    """The 16-bit model with keys and values replaced by x8 * scale on entering the cache: every append is followed by
    the quantise-dequantise round trip of the positions it wrote (the prefill's attention reads them from the cache)."""
    from mm_interleaved_b200 import ops
    append = ops.rope_qk_append_

    def quantised(q, k, v, cos, sin, pos, kc, vc, slot):
        append(q, k, v, cos, sin, pos, kc, vc, slot)
        s = int(slot)
        for c in (kc, vc):
            x = c[:, s:s + q.shape[1]]
            x8, sc = ops.quantize_kv_fp8(x)
            x.copy_((x8.float() * sc[..., None]).to(x.dtype))
    monkeypatch.setattr(ops, "rope_qk_append_", quantised)


def _chunked_logits(model, embeds, mask, pos, chunks, kv_fp8, vision=None, cross=None):
    """The positions fed in chunks over one static cache: (B, L, V) logits of every position."""
    B, L, _ = embeds.shape
    past = model.mm_decoder.static_cache(B, L, kv_fp8=kv_fp8)
    out = []
    with torch.no_grad():
        for a, b in zip(chunks[:-1], chunks[1:]):
            h = model.mm_decoder(inputs_embeds=embeds[:, a:b], attention_mask=mask[:, :b], position_ids=pos[:, a:b],
                                 past_key_values=past, vision_hidden_states=vision,
                                 cross_attention_mask=None if cross is None else cross[:, a:b], use_cache=True,
                                 return_dict=True).last_hidden_state
            out.append(model.text_decoder.logits(h).float())
    return torch.cat(out, 1)


def _assert_close(got, want):
    err = (got - want).abs().max().item()
    assert err <= 3e-2 * want.abs().max().item(), f"max |diff| {err} against max |logit| {want.abs().max().item()}"


def _tiny():
    from tests.test_fp8_decode_gpu import _tiny as tiny
    return tiny()


def test_tiny_decoder_fp8_cache_equals_the_16_bit_model_on_x8_scale(monkeypatch):
    from mm_interleaved_b200 import ops
    dev, ids, nimg, vis_d = _tiny()
    mm_embeds, cross, feats = dev.prepare(ids, vis_d, nimg, 2)
    mask = torch.ones_like(ids)
    mask[0, :2] = 0
    pos = (mask.cumsum(-1) - 1).masked_fill(mask == 0, 1)
    vision = dev.mm_decoder.prepare_vision(feats)
    L = ids.shape[1]
    plans = [list(range(L + 1)), [0, L - 3] + list(range(L - 2, L + 1)), [0, 4, L - 2, L - 1, L]]   # steps; prefill;
    calls = {}                                                                                         # chunks
    for name in ("rope_qk_append_fp8_", "attention_decode_fp8", "kv_dequantize_fp8"):
        fn = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _f=fn, _n=name, **k: calls.__setitem__(_n, calls.get(_n, 0) + 1) or _f(*a, **k))
    got = [_chunked_logits(dev, mm_embeds, mask, pos, c, True, vision, cross) for c in plans]
    assert set(calls) == {"rope_qk_append_fp8_", "attention_decode_fp8", "kv_dequantize_fp8"}
    plain = _chunked_logits(dev, mm_embeds, mask, pos, plans[0], False, vision, cross)
    _quantise_on_entry(monkeypatch)
    for c, g in zip(plans, got):
        want = _chunked_logits(dev, mm_embeds, mask, pos, c, False, vision, cross)
        _assert_close(g[:, 2:], want[:, 2:])                                # row 0's padded positions see no key
    assert not torch.equal(plain, got[0])


def test_13b_width_layers_fp8_cache_equals_the_16_bit_model_on_x8_scale(monkeypatch):
    from mm_interleaved_b200 import LlamaMMFSConfig
    from mm_interleaved_b200.mm_interleaved import InterleavedForward
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = InterleavedForward(LlamaMMFSConfig(num_hidden_layers=2), orig_vocab_size=32000)
    model = model.to(BF16).eval()
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0.0, 0.02)
        for layer in model.mm_decoder.layers:
            layer.input_layernorm.weight.fill_(1.0)
            layer.post_attention_layernorm.weight.fill_(1.0)
        model.mm_decoder.norm.weight.fill_(1.0)
    B, L = 4, 300
    embeds = torch.randn(B, L, 5120, device="cuda").to(BF16)
    mask = torch.ones(B, L, dtype=torch.long, device="cuda")
    pos = mask.cumsum(-1) - 1
    chunks = [0, L - 4, L - 3, L - 2, L - 1, L]
    got = _chunked_logits(model, embeds, mask, pos, chunks, True)
    _quantise_on_entry(monkeypatch)
    want = _chunked_logits(model, embeds, mask, pos, chunks, False)
    _assert_close(got, want)


@pytest.mark.parametrize("num_beams", [1, 3])
def test_graphed_fp8_cache_decoding_equals_eager(num_beams):
    from mm_interleaved_b200.generation import BeamDecoder, TokenDecoder
    dev, ids, nimg, vis_d = _tiny()
    dev.enable_fp8_kv_cache()
    kw = dict(max_new_tokens=7, eos_token_id=[2, 17], min_length=3, num_beams=num_beams)
    eager = dev.generate_texts(ids, vis_d, nimg, 2, **kw).cpu()
    dev.enable_decode_graphs()
    graphed = dev.generate_texts(ids, vis_d, nimg, 2, **kw).cpu()
    (dec,) = dev._decode_graphs.values()
    assert torch.equal(graphed, eager), (graphed, eager)
    if num_beams == 1:
        assert isinstance(dec, TokenDecoder) and all(c.k.dtype == torch.float8_e4m3fn for c in dec.past)
    else:
        assert isinstance(dec, BeamDecoder) and dec.gen.dtype == torch.float8_e4m3fn and dec.gen_scale is not None
    dev.enable_fp8_kv_cache(False)
    assert dev._decode_graphs == {}
    plain = dev.generate_texts(ids, vis_d, nimg, 2, **kw).cpu()
    (dec,) = dev._decode_graphs.values()
    assert all(t.dtype == BF16 for t in ([dec.gen] if num_beams > 1 else [c.k for c in dec.past]))
    assert plain.shape[0] == eager.shape[0]


def test_interleaved_session_beam_turn_equals_the_call_without_a_session():
    from tests.test_interleaved_gpu import GEN, build, sample
    model = build()
    model.enable_decode_graphs().enable_fp8_kv_cache()
    inputs = sample()
    gen = dict(GEN, num_beams=5, max_length=5)
    kw = {k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors", "num_image_per_seq")}
    out = model.generate_interleaved(**kw, num_iter=1, return_session=True, **gen)
    assert out["session"].cache[0].k.dtype == torch.float8_e4m3fn
    alone = model.generate(mode="generate_texts", **{k: v.clone() for k, v in inputs.items()}, **gen)["text_ids"]
    assert torch.equal(out["turns"][0]["text_ids"].cpu(), alone.cpu()), (out["turns"][0]["text_ids"], alone)


def test_cache_bytes_at_13b_widths_about_halve():
    """2 layers of 40 x 128 heads, B = 4, 5 beams, a 2048-token prompt: the graphed beam decoder's cache (prompt prefix,
    generated positions, scales) against the 16-bit one."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.generation import BeamDecoder
    from mm_interleaved_b200.mm_interleaved import InterleavedForward
    torch.manual_seed(0)
    cfg = m.LlamaMMFSConfig(num_hidden_layers=2, vocab_size=32002)
    with torch.device("cuda"):
        model = InterleavedForward(cfg, special_tokens=dict(bos_token_id=1, image_token_id=32000, soi_token_id=32001),
                                   orig_vocab_size=32000).to(BF16).eval()
    B, L, nb, max_new, n_tok = 4, 2048, 5, 20, 64
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, 31999, (B, L), generator=g)
    ids[:, 0] = 1
    for i in range(4):
        ids[:, 10 + 300 * i] = 32001
        ids[:, 11 + 300 * i:11 + 300 * i + n_tok] = 32000
    nimg = torch.full((B,), 4, dtype=torch.long)
    vis = {"vis_embed": torch.randn((4 * B, n_tok, cfg.hidden_size), generator=g).to(BF16).cuda() * 0.1,
           "multiscale_features": [torch.randn((4 * B, cfg.image_embed_dim, s, s), generator=g).to(BF16).cuda()
                                   for s in cfg.spatial_shapes]}
    model.enable_decode_graphs()
    sizes = {}
    for fp8 in (False, True):
        model.enable_fp8_kv_cache(fp8)
        with torch.no_grad():
            out = model.generate_texts(ids.cuda(), vis, nimg.cuda(), 4, max_new_tokens=max_new, eos_token_id=[2],
                                       min_length=8, num_beams=nb)
        assert out.shape[0] == B
        (dec,) = model._decode_graphs.values()
        assert isinstance(dec, BeamDecoder)
        sizes[fp8] = sum(t.numel() * t.element_size() for t in (dec.prefix, dec.gen, dec.prefix_scale, dec.gen_scale)
                         if t is not None)
    assert sizes[True] <= 0.53 * sizes[False], sizes
