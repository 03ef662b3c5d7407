"""GPU tests of FP8 decoding: ``ops.linear_fp8`` against float64 at the decoder's shapes, its determinism and graph
capture, and the model switch (``enable_fp8_decode``) against the 16-bit model whose weights are replaced by the
quantised ``w8 * scale``, eagerly and graphed."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.golden.make_golden import LLAMA_TINY  # noqa: E402

BF16, F16 = torch.bfloat16, torch.float16
# (N, K): fused QKV, o_proj, fused gate/up, down_proj, the folded head (32002 padded to 32128) at the 13B widths; an N
# tail that is not a tile multiple with a K that leaves a short last stage; a tiny one
SHAPES = [(15360, 5120), (5120, 5120), (27648, 5120), (5120, 13824), (32128, 5120), (1000, 272), (70, 16)]
MS = [1, 2, 5, 16, 20, 64]


def _case(M, N, K, dtype, seed, bias=True, residual=True):
    from mm_interleaved_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn((N, K), generator=g, device="cuda") * torch.rand((N, 1), generator=g, device="cuda") * 0.05
    w8, s = ops.quantize_fp8_per_channel(w)
    x = torch.randn((M, K), generator=g, device="cuda").to(dtype)
    b = torch.randn((N,), generator=g, device="cuda").to(dtype) if bias else None
    r = torch.randn((M, N), generator=g, device="cuda").to(dtype) if residual else None
    return x, w8, s, b, r


def _ref(x, w8, s, b, r):
    wq = w8.double() * s.double()[:, None]
    prod = x.double() @ wq.t()
    mag = x.double().abs() @ wq.abs().t()
    if b is not None:
        prod = prod + b.double()
    if r is not None:
        prod = prod + r.double()
    return prod, mag


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("N, K", SHAPES)
def test_linear_fp8_against_float64(N, K, dtype):
    from mm_interleaved_b200 import ops
    u = 2.0 ** -8 if dtype == BF16 else 2.0 ** -11                 # one rounding of the output
    for i, M in enumerate(MS):
        x, w8, s, b, r = _case(M, N, K, dtype, seed=1000 * i + N % 997, bias=i % 2 == 0, residual=i % 3 != 2)
        assert ops.linear_fp8_supported(x, w8)
        y = ops.linear_fp8(x, w8, s, b, r)
        ref, mag = _ref(x, w8, s, b, r)
        err = (y.double() - ref).abs()
        tol = u * ref.abs() + K * 2.0 ** -24 * mag + 1e-6           # + fp32 summation over K
        bad = err > tol
        assert not bool(bad.any()), f"M={M}: {int(bad.sum())} outside, worst {float((err - tol).max())}"
        assert torch.equal(ops.linear_fp8(x, w8, s, b, r), y), f"M={M}: two runs differ"


def test_linear_fp8_in_place_residual_and_graph_replay():
    from mm_interleaved_b200 import ops
    x, w8, s, b, r = _case(5, 5120, 13824, BF16, seed=7)
    want = ops.linear_fp8(x, w8, s, b, r)
    acc = r.clone()
    assert ops.linear_fp8(x, w8, s, b, acc, out=acc) is acc and torch.equal(acc, want)
    static_x = x.clone()
    out = torch.empty_like(want)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.linear_fp8(static_x, w8, s, b, r, out=out)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.linear_fp8(static_x, w8, s, b, r, out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    x2 = torch.randn_like(x)
    static_x.copy_(x2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ops.linear_fp8(x2, w8, s, b, r))


def test_linear_fp8_refusals_come_from_the_library():
    from mm_interleaved_b200 import ops
    x, w8, s, _, _ = _case(65, 64, 64, BF16, seed=3, bias=False, residual=False)
    assert not ops.linear_fp8_supported(x, w8)
    with pytest.raises(RuntimeError, match=r"unsupported \(-2\).*M <= 64"):
        ops.linear_fp8(x, w8, s)
    x, w8, s, _, _ = _case(2, 64, 24, BF16, seed=3, bias=False, residual=False)
    assert not ops.linear_fp8_supported(x, w8)
    with pytest.raises(RuntimeError, match=r"unsupported \(-2\).*multiple of 16"):
        ops.linear_fp8(x, w8, s)


# ---- the model switch ------------------------------------------------------------------------------------------------
def _quantised_copy(model):
    """The same model with every FP8-routed weight (fused QKV, fused gate/up, the folded head) replaced in place by its
    ``w8 * scale`` (bf16, exact)."""
    from mm_interleaved_b200 import ops
    q = copy.deepcopy(model)
    with torch.no_grad():
        for layer in q.mm_decoder.layers:
            a, m = layer.self_attn, layer.mlp
            for lin in (a.q_proj, a.k_proj, a.v_proj, m.gate_proj, m.up_proj):
                w8, s = ops.quantize_fp8_per_channel(lin.weight)
                lin.weight.copy_(w8.float() * s[:, None])
        td = q.text_decoder
        w, _ = td._fused()
        w8, s = ops.quantize_fp8_per_channel(w)
        td.head.weight.copy_((w8.float() * s[:, None])[:td.head.weight.shape[0]])
        td.head_new.weight.zero_()                                  # the fold adds it to the tail rows: already in
    return q


def _teacher_forced_logits(model, embeds, mask, pos, vision=None, cross=None):
    """Every position fed as its own decode step over a static cache: (B, L, V) logits."""
    B, L, _ = embeds.shape
    past = model.mm_decoder.static_cache(B, L)
    out = []
    with torch.no_grad():
        for t in range(L):
            h = model.mm_decoder(inputs_embeds=embeds[:, t:t + 1], attention_mask=mask[:, :t + 1],
                                 position_ids=pos[:, t:t + 1], past_key_values=past, vision_hidden_states=vision,
                                 cross_attention_mask=None if cross is None else cross[:, t:t + 1], use_cache=True,
                                 return_dict=True).last_hidden_state
            out.append(model.text_decoder.logits(h).float())
    return torch.cat(out, 1)


def _tiny():
    from tests.test_generate_gpu import _setup
    cfg, dev, sd, ids, nimg, vis, vis_d = _setup()
    dev = dev.to(BF16)
    vis_d = {"vis_embed": vis_d["vis_embed"].to(BF16), "multiscale_features": [f.to(BF16) for f in vis_d["multiscale_features"]]}
    return dev, ids.cuda(), nimg.cuda(), vis_d


def _assert_close(got, want):
    err = (got - want).abs().max().item()
    assert err <= 3e-2 * want.abs().max().item(), f"max |diff| {err} against max |logit| {want.abs().max().item()}"


def test_tiny_decoder_fp8_steps_equal_the_quantised_16_bit_model():
    from mm_interleaved_b200 import ops
    dev, ids, nimg, vis_d = _tiny()
    ref_model = _quantised_copy(dev)
    dev.enable_fp8_decode()
    mm_embeds, cross, feats = dev.prepare(ids, vis_d, nimg, 2)
    mask = torch.ones_like(ids)
    pos = (mask.cumsum(-1) - 1)
    before = ops.launch_counter[0]
    got = _teacher_forced_logits(dev, mm_embeds, mask, pos, dev.mm_decoder.prepare_vision(feats), cross)
    assert ops.launch_counter[0] > before
    want = _teacher_forced_logits(ref_model, mm_embeds, mask, pos, ref_model.mm_decoder.prepare_vision(feats), cross)
    _assert_close(got, want)
    plain = _teacher_forced_logits(dev.enable_fp8_decode(False), mm_embeds, mask, pos,
                                   dev.mm_decoder.prepare_vision(feats), cross)
    assert not torch.equal(plain, got)                              # the switch changed the weights the steps read


def test_13b_width_layers_fp8_steps_equal_the_quantised_16_bit_model():
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
    ref_model = _quantised_copy(model)
    model.enable_fp8_decode()
    B, L = 5, 6
    embeds = (torch.randn(B, L, 5120, device="cuda")).to(BF16)
    mask = torch.ones(B, L, dtype=torch.long, device="cuda")
    pos = mask.cumsum(-1) - 1
    got = _teacher_forced_logits(model, embeds, mask, pos)
    want = _teacher_forced_logits(ref_model, embeds, mask, pos)
    _assert_close(got, want)


@pytest.mark.parametrize("num_beams", [1, 2])              # 2 prompts x 2 beams: 4 rows, within FP8_DECODE_MAX_ROWS
def test_graphed_fp8_decoding_equals_eager_fp8(num_beams):
    dev, ids, nimg, vis_d = _tiny()
    dev.enable_fp8_decode()
    kw = dict(max_new_tokens=7, eos_token_id=[2, 17], min_length=3, num_beams=num_beams)
    eager = dev.generate_texts(ids, vis_d, nimg, 2, **kw).cpu()
    dev.enable_decode_graphs()
    graphed = dev.generate_texts(ids, vis_d, nimg, 2, **kw).cpu()
    assert len(dev._decode_graphs) == 1
    assert torch.equal(graphed, eager), (graphed, eager)
    dev.enable_fp8_decode(False)                                    # drops the FP8 graph
    assert dev._decode_graphs == {}
    dev.enable_decode_graphs(False)
