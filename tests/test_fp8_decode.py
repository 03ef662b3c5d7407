"""CPU tests of FP8 decoding: the per-channel E4M3 quantiser, the argument refusals of ``ops.linear_fp8``, and which
calls ``decode_linear`` routes to it (the kernels are replaced by stand-ins that log the call, as in
test_training_switch.py)."""
import pytest
import torch
import torch.nn.functional as F

from mm_interleaved_b200 import llama_mmfs, ops
from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, decode_linear
from mm_interleaved_b200.mm_interleaved import InterleavedForward, TextDecoder
from mm_interleaved_b200._cache import WeightCache

BF16 = torch.bfloat16


def _weights(seed=0):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn((48, 96), generator=g) * torch.logspace(-6, 4, 48)[:, None]   # rows over ten decades
    w[7] = 0.0
    w[11, :5] = 0.0
    w[13] = torch.randn(96, generator=g) * 1e-30                                  # tiny: zero rows in fp16
    return w


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_quantiser(dtype):
    w = _weights().to(dtype)
    if dtype != torch.float32:
        w = torch.nan_to_num(w, posinf=0.0, neginf=0.0)
    w8, s = ops.quantize_fp8_per_channel(w)
    assert w8.dtype == torch.float8_e4m3fn and w8.shape == w.shape and s.dtype == torch.float32 and s.shape == (48,)
    m, e = torch.frexp(s)
    assert bool((m == 0.5).all()), "every scale is a power of two"
    wf = w.float()
    amax = wf.abs().amax(1)
    assert bool((s[amax == 0] == 1).all()), "an all-zero row has scale 1"
    assert bool(((wf / s[:, None]).abs() <= 448).all())
    nz = amax > 0
    assert bool((amax[nz] / s[nz] > 224).all()), "the least power of two: the row's largest entry lands in (224, 448]"
    wq = w8.float() * s[:, None]
    assert torch.equal(wq.to(torch.bfloat16).float(), wq), "w8 * s is exact in bf16"
    # round to nearest: half an e4m3 ulp at the entry's magnitude (3 mantissa bits; subnormal below 2^-6 * s)
    err = (wq - wf).abs()
    bound = torch.where(wf.abs() >= 2.0 ** -6 * s[:, None], 2.0 ** -4 * wf.abs(), 2.0 ** -10 * s[:, None].expand_as(wf))
    assert bool((err <= bound).all())


def test_quantiser_matches_round_to_nearest_even():
    w = _weights(1)
    w8, s = ops.quantize_fp8_per_channel(w)
    assert torch.equal(w8.view(torch.uint8), (w / s[:, None]).to(torch.float8_e4m3fn).view(torch.uint8))


def test_quantiser_refuses():
    with pytest.raises(RuntimeError, match="2-D"):
        ops.quantize_fp8_per_channel(torch.zeros(4, 4, 4))
    with pytest.raises(RuntimeError, match="2-D"):
        ops.quantize_fp8_per_channel(torch.zeros(4, 4, dtype=torch.float64))


def _fp8_args(M=2, N=32, K=64, dtype=BF16):
    w8, s = ops.quantize_fp8_per_channel(torch.randn(N, K))
    return torch.randn(M, K).to(dtype), w8, s


@pytest.mark.parametrize("case, match", [
    ("cpu", "CUDA bf16 / fp16"),
    ("fp32", "CUDA bf16 / fp16"),
])
def test_linear_fp8_refuses_x(case, match):
    x, w8, s = _fp8_args(dtype=torch.float32 if case == "fp32" else BF16)
    with pytest.raises(RuntimeError, match=match):
        ops.linear_fp8(x, w8, s)


def test_linear_fp8_refuses_recording():
    x, w8, s = _fp8_args()
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.linear_fp8(x.requires_grad_(), w8, s)


def test_linear_fp8_supported():
    x, w8, s = _fp8_args()
    assert not ops.linear_fp8_supported(x, w8)                                      # a CPU tensor
    meta = lambda *shape, dt=BF16: torch.empty(shape, dtype=dt, device="meta")
    w = meta(32, 64, dt=torch.float8_e4m3fn)
    assert not ops.linear_fp8_supported(meta(2, 64), w)                             # not CUDA either
    assert not ops.linear_fp8_supported(meta(2, 64), meta(32, 64))


# ---- routing ---------------------------------------------------------------------------------------------------------
def _stand_ins(monkeypatch, calls):
    """ops kernels as torch stand-ins; ``linear_fp8`` logs its (rows, N, K) and computes the 16-bit result of w8 * s."""
    def linear_fp8(x, w8, scale, bias=None, residual=None, out=None):
        calls.append((x.numel() // x.shape[-1], w8.shape[0], w8.shape[1]))
        y = F.linear(x.float(), w8.float() * scale[:, None], None if bias is None else bias.float())
        if residual is not None:
            y = y + residual.float()
        y = y.to(x.dtype)
        return y if out is None else out.copy_(y)
    monkeypatch.setattr(ops, "linear_fp8", linear_fp8)
    monkeypatch.setattr(ops, "rmsnorm", lambda x, w, eps: (x.float() * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype) * w)
    monkeypatch.setattr(ops, "swiglu", lambda gu: F.silu(gu[..., :gu.shape[-1] // 2]) * gu[..., gu.shape[-1] // 2:])
    monkeypatch.setattr(ops, "rope_qk_", lambda q, k, cos, sin, pos: None)
    monkeypatch.setattr(ops, "attention", lambda q, k, v, key_mask=None, causal=True, past=0: v[:, -q.shape[1]:].reshape(
        q.shape[0], q.shape[1], -1).contiguous())


CFG = dict(vocab_size=40, hidden_size=32, intermediate_size=48, num_hidden_layers=2, num_attention_heads=2,
           max_position_embeddings=64, cross_attention_frequency=8, spatial_shapes=[2], image_embed_dim=16)


def _tiny_model():
    torch.manual_seed(0)
    m = InterleavedForward(LlamaMMFSConfig(**CFG), orig_vocab_size=38).to(BF16).eval()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _decoder_calls(model, T, B=2, grad=False, calls=None):
    x = torch.randn(B, T, CFG["hidden_size"]).to(BF16)
    before = len(calls)
    with torch.set_grad_enabled(grad):
        if grad:
            x.requires_grad_()
        h = model.mm_decoder(inputs_embeds=x, use_cache=False, return_dict=True).last_hidden_state
        if not grad:
            model.text_decoder.logits(h)
    return calls[before:]


def test_switch_off_never_calls_linear_fp8(monkeypatch):
    calls = []
    _stand_ins(monkeypatch, calls)
    model = _tiny_model()
    for T in (1, 5):
        assert _decoder_calls(model, T, calls=calls) == []
    model.enable_fp8_decode(True).enable_fp8_decode(False)
    assert _decoder_calls(model, 1, calls=calls) == []


def test_switch_on_routes_decode_steps_only(monkeypatch):
    calls = []
    _stand_ins(monkeypatch, calls)
    model = _tiny_model().enable_fp8_decode()
    C, I, Vp = CFG["hidden_size"], CFG["intermediate_size"], 128
    per_layer = [(2, 3 * C, C), (2, 2 * I, C)]                  # qkv, gate/up; not o_proj and down_proj (N < 2K)
    assert _decoder_calls(model, 1, calls=calls) == per_layer * CFG["num_hidden_layers"] + [(2, Vp, C)]
    assert _decoder_calls(model, 5, calls=calls) == []                              # the prefill
    rows = llama_mmfs.FP8_DECODE_MAX_ROWS
    assert len(_decoder_calls(model, 1, B=rows, calls=calls)) == 2 * CFG["num_hidden_layers"] + 1
    assert _decoder_calls(model, 1, B=rows + 1, calls=calls) == []                  # more rows than where it wins


def test_switch_on_leaves_recording_calls_alone(monkeypatch):
    calls = []
    _stand_ins(monkeypatch, calls)
    w = torch.randn(64, CFG["hidden_size"]).to(BF16)
    x = torch.randn(2, 1, CFG["hidden_size"]).to(BF16).requires_grad_()
    y = decode_linear(x, w, WeightCache(), "w")
    assert calls == [] and y.requires_grad
    with torch.no_grad():
        decode_linear(x, w, WeightCache(), "w")
    assert calls == [(2, 64, CFG["hidden_size"])]


def test_forward_stays_16_bit(monkeypatch):
    """``InterleavedForward.forward`` over a prompt: the decoder and the head see every position, never one."""
    calls = []
    _stand_ins(monkeypatch, calls)
    model = _tiny_model().enable_fp8_decode()
    monkeypatch.setattr(model, "prepare", lambda *a: (torch.randn(2, 6, CFG["hidden_size"]).to(BF16), None, None))
    with torch.no_grad():
        logits = model.forward(None, None, None, 0)
    assert logits.shape == (2, 6, CFG["vocab_size"]) and calls == []


def test_decode_linear_matches_the_16_bit_model_on_wq(monkeypatch):
    """With the stand-in computing x @ (w8 * s)^T, the FP8 route equals the 16-bit route on weights w8 * s."""
    calls = []
    _stand_ins(monkeypatch, calls)
    w = torch.randn(72, 32).to(BF16)
    b = torch.randn(72).to(BF16)
    r = torch.randn(3, 1, 72).to(BF16)
    x = torch.randn(3, 1, 32).to(BF16)
    w8, s = ops.quantize_fp8_per_channel(w)
    wq = (w8.float() * s[:, None]).to(BF16)
    with torch.no_grad():
        got = decode_linear(x, w, WeightCache(), "w", residual=r.clone())
        ref = decode_linear(x, wq, None, "w", residual=r.clone())
        assert torch.allclose(got.float(), ref.float(), atol=1e-2, rtol=1e-2)
        assert torch.equal(decode_linear(x, w, WeightCache(), "w", bias=b),
                           (F.linear(x.float(), wq.float(), b.float())).to(BF16))
        into = r.clone()
        assert decode_linear(x, w, WeightCache(), "w", residual=into, inplace=True) is into


def test_fp8_copies_are_cached_per_weight(monkeypatch):
    calls, built = [], []
    _stand_ins(monkeypatch, calls)
    quant = ops.quantize_fp8_per_channel
    monkeypatch.setattr(ops, "quantize_fp8_per_channel", lambda w: built.append(w.shape) or quant(w))
    model = _tiny_model().enable_fp8_decode()
    _decoder_calls(model, 1, calls=calls)
    _decoder_calls(model, 1, calls=calls)
    assert len(built) == 2 * CFG["num_hidden_layers"] + 1                            # once per weight
    with torch.no_grad():
        model.mm_decoder.layers[0].mlp.up_proj.weight.mul_(2)
    _decoder_calls(model, 1, calls=calls)
    assert len(built) == 2 * CFG["num_hidden_layers"] + 2                            # rebuilt when its source changes


def test_toggling_drops_captured_decode_graphs():
    model = _tiny_model().enable_decode_graphs()
    for enabled in (True, False):
        model._decode_graphs["captured"] = object()
        model.enable_fp8_decode(enabled)
        assert model._decode_graphs == {}
    no_graphs = _tiny_model().enable_fp8_decode()
    assert no_graphs._decode_graphs is None
    on = [m._fp8 is not None for m in model.modules() if isinstance(m, (llama_mmfs.LlamaAttention, llama_mmfs.LlamaMLP,
                                                                        TextDecoder))]
    assert len(on) == 2 * CFG["num_hidden_layers"] + 1 and not any(on)
    assert all(m._fp8 is not None for m in no_graphs.modules()
               if isinstance(m, (llama_mmfs.LlamaAttention, llama_mmfs.LlamaMLP, TextDecoder)))
