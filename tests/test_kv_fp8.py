"""CPU tests of the FP8 KV cache: the per-head E4M3 quantiser, the argument refusals of the four kernels' wrappers and
entry points, and which ops each generation path calls with ``enable_fp8_kv_cache`` off and on (the kernels are
replaced by torch stand-ins that log the call, as in test_fp8_decode.py)."""
import pytest
import torch
import torch.nn.functional as F

from mm_interleaved_b200 import generation, llama_mmfs, ops
from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, PreparedVision, StaticKV
from mm_interleaved_b200.mm_interleaved import InterleavedForward

BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn


def _keys(seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((3, 5, 6, 32), generator=g) * torch.logspace(-8, 6, 6)[:, None]   # heads over fourteen decades
    x[0, 1, 2] = 0.0
    x[1, 2, 3, :7] = 0.0
    x[2, 4, 1] = 448.0                                                                  # exactly at the range: scale 1
    x[2, 3, 1] = 0.1
    x[2, 3, 1, 0] = 450.0                                                               # just above: scale 2
    return x


@pytest.mark.parametrize("dtype", [torch.float32, BF16, torch.float16])
def test_quantiser_properties(dtype):
    x = _keys().to(dtype)
    if dtype == torch.float16:
        x = torch.nan_to_num(x, posinf=0.0, neginf=0.0)
    x8, s = ops.quantize_kv_fp8(x)
    assert x8.dtype == E4M3 and x8.shape == x.shape and s.dtype == torch.float32 and s.shape == x.shape[:-1]
    m, _ = torch.frexp(s)
    assert bool((m == 0.5).all()), "every scale is a power of two"
    xf = x.float()
    amax = xf.abs().amax(-1)
    assert bool((s[amax == 0] == 1).all()), "an all-zero vector has scale 1"
    assert bool(((xf / s[..., None]).abs() <= 448).all())
    nz = amax > 0
    assert bool((amax[nz] / (s[nz] / 2) > 448).all()), "the least such power of two"
    assert float(s[2, 4, 1]) == 1.0 and float(s[2, 3, 1]) == 2.0
    xq = x8.float() * s[..., None]
    assert torch.equal(xq.to(BF16).float(), xq), "x8 * scale is exact in bf16"
    big = (s >= 2.0 ** -15) & (amax <= 57344)               # within fp16: its subnormal step 2^-24 is 2^-9 * 2^-15
    assert torch.equal(xq[big].to(torch.float16).float(), xq[big]), "and in fp16 within its normal range"


def test_quantiser_rounds_to_nearest_even():
    """Against a float64 rounding to the e4m3 grid (3 mantissa bits, subnormal step 2^-9), ties to even."""
    x = _keys(1)
    x8, s = ops.quantize_kv_fp8(x)
    y = (x.double() / s.double()[..., None])
    e = torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -6)))
    step = torch.exp2(e - 3)                                                # the grid spacing at |y|
    r = torch.round(y / step) * step                                        # torch.round: half to even
    assert torch.equal(x8.double(), r)


def test_quantiser_refuses():
    with pytest.raises(RuntimeError, match="H, hd"):
        ops.quantize_kv_fp8(torch.zeros(4))
    with pytest.raises(RuntimeError, match="H, hd"):
        ops.quantize_kv_fp8(torch.zeros(4, 4, dtype=torch.float64))


def test_scale_rows_are_whole_16_byte_rows():
    assert [ops.kv_scale_heads(h) for h in (1, 2, 4, 5, 40)] == [4, 4, 4, 8, 40]


# ---- refusals --------------------------------------------------------------------------------------------------------
def _fp8_cache(B=2, T=8, H=2, hd=64):
    return (torch.zeros((B, T, H, hd), dtype=E4M3), torch.zeros((B, T, H, hd), dtype=E4M3),
            torch.ones((B, T, 4)), torch.ones((B, T, 4)))


def test_wrappers_refuse_cpu_and_fp64_tensors():
    k8, v8, ks, vs = _fp8_cache()
    q = torch.zeros((2, 1, 2, 64), dtype=BF16)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.attention_decode_fp8(q, k8, v8, ks, vs)
    with pytest.raises(RuntimeError, match="fp32 / bf16 / fp16"):
        ops.attention_decode_fp8(q.double(), k8, v8, ks, vs)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.attention_decode_shared_fp8(q, k8[:1], v8[:1], ks[:1], vs[:1], k8, v8, ks, vs, torch.zeros(1, dtype=torch.long))
    with pytest.raises(RuntimeError, match="float8_e4m3fn CUDA"):
        ops.kv_dequantize_fp8(k8, ks, BF16)
    with pytest.raises(RuntimeError, match="fp32 / bf16 / fp16"):
        ops.kv_dequantize_fp8(k8, ks, torch.float64)
    qkv = torch.zeros((2, 1, 3, 2, 64), dtype=BF16)
    cos = torch.zeros((16, 64))
    args = (cos, cos, torch.zeros(1, dtype=torch.long), k8, v8, ks, vs, 0)
    with pytest.raises(RuntimeError, match="fp32 / bf16 / fp16"):
        ops.rope_qk_append_fp8_(qkv[:, :, 0].double(), qkv[:, :, 1].double(), qkv[:, :, 2].double(), *args)
    with pytest.raises(RuntimeError, match="dense heads"):
        ops.rope_qk_append_fp8_(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], *args)


def test_wrappers_refuse_recording():
    k8, v8, ks, vs = _fp8_cache()
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.attention_decode_fp8(torch.zeros((2, 1, 2, 64), dtype=BF16, requires_grad=True), k8, v8, ks, vs)


# fake, never dereferenced device addresses: every call below is refused before a launch
A = [0x10000 * (i + 1) for i in range(13)]


def _decode(**over):
    from mm_interleaved_b200 import _lib
    H, hd, T = 2, 128, 64
    a = dict(q=A[0], k=A[1], v=A[2], ks=A[3], vs=A[4], out=A[5], mask=A[6], scratch=A[7], B=2, H=H, Tkv=T, hd=hd,
             q_bs=3 * H * hd, kv_bs=T * H * hd, kv_ts=H * hd, s_bs=T * 4, s_ts=4, o_bs=H * hd, scale=0.125, causal=1,
             past=T - 1, dtype=_lib.BF16)
    a.update(over)
    rc = _lib.lib().mmfs_attn_decode_fp8(*a.values(), None)
    return rc, _lib.lib().mmfs_last_error().decode()


def _shared(**over):
    from mm_interleaved_b200 import _lib
    H, hd, Tp, mn = 2, 64, 32, 4
    a = dict(q=A[0], kp=A[1], vp=A[2], ksp=A[3], vsp=A[4], kg=A[5], vg=A[6], ksg=A[7], vsg=A[8], out=A[9], mask=A[10],
             plen=A[11], scratch=A[12], R=6, G=3, H=H, Tkv=Tp + mn, Tp=Tp, max_new=mn, hd=hd, q_bs=3 * H * hd,
             p_bs=Tp * H * hd, p_ts=H * hd, ps_bs=Tp * 4, ps_ts=4, g_bs=mn * H * hd, g_ts=H * hd, gs_bs=mn * 4, gs_ts=4,
             o_bs=H * hd, scale=0.125, causal=1, past=Tp + mn - 1, dtype=_lib.BF16)
    a.update(over)
    rc = _lib.lib().mmfs_attn_decode_shared_fp8(*a.values(), None)
    return rc, _lib.lib().mmfs_last_error().decode()


def _append(**over):
    from mm_interleaved_b200 import _lib
    H, hd = 2, 64
    a = dict(q=A[0], k=A[1], v=A[2], cos=A[3], sin=A[4], pos=A[5], kc=A[6], vc=A[7], ks=A[8], vs=A[9], slot_dev=None,
             slot=0, n=4, T=2, H=H, hd=hd, qs=3 * H * hd, kst=3 * H * hd, vst=3 * H * hd, c_bs=8 * H * hd, c_ts=H * hd,
             s_bs=32, s_ts=4, ppb=0, dtype=_lib.BF16)
    a.update(over)
    rc = _lib.lib().mmfs_rope_qk_append_fp8(*a.values(), None)
    return rc, _lib.lib().mmfs_last_error().decode()


def _dequant(**over):
    from mm_interleaved_b200 import _lib
    a = dict(x=A[0], s=A[1], out=A[2], B=2, T=4, H=2, hd=64, x_bs=512, x_ts=128, s_bs=16, s_ts=4, o_bs=512, o_ts=128,
             dtype=_lib.BF16)
    a.update(over)
    rc = _lib.lib().mmfs_kv_dequantize_fp8(*a.values(), None)
    return rc, _lib.lib().mmfs_last_error().decode()


@pytest.mark.parametrize("call, over, code, match", [
    (_decode, dict(k=None), -1, "null pointer"),
    (_decode, dict(hd=0), -1, "bad shape"),
    (_decode, dict(past=-1), -1, "negative past"),
    (_decode, dict(hd=48), -2, "hd % 32"),
    (_decode, dict(hd=288), -2, "hd % 32"),
    (_decode, dict(kv_ts=200), -2, "aligned"),
    (_decode, dict(v=A[2] + 8), -2, "aligned"),
    (_decode, dict(s_ts=1), -2, ">= H"),
    (_decode, dict(dtype=3), -2, "dtype"),
    (_shared, dict(R=7), -1, "whole groups"),
    (_shared, dict(max_new=0), -1, "max_new"),
    (_shared, dict(vsg=None), -1, "null pointer"),
    (_shared, dict(g_ts=100), -2, "aligned"),
    (_shared, dict(dtype=3), -2, "dtype"),
    (_append, dict(ks=None), -1, "null pointer"),
    (_append, dict(H=0), -1, "bad shape"),
    (_append, dict(hd=63), -2, "even head dim"),
    (_append, dict(s_ts=1), -2, "H heads"),
    (_append, dict(dtype=3), -2, "dtype"),
    (_dequant, dict(out=None), -1, "null pointer"),
    (_dequant, dict(hd=24), -2, "hd % 16"),
    (_dequant, dict(x_ts=8), -2, "aligned"),
])
def test_entry_points_refuse_with_codes(call, over, code, match):
    rc, msg = call(**over)
    assert rc == code and match in msg, (rc, msg)


def test_empty_calls_are_no_ops():
    assert _decode(B=0, q=None)[0] == 0
    assert _shared(R=0, q=None)[0] == 0
    assert _append(n=0, q=None)[0] == 0
    assert _dequant(T=0, x=None)[0] == 0


# ---- routing ---------------------------------------------------------------------------------------------------------
CFG = dict(vocab_size=40, hidden_size=32, intermediate_size=48, num_hidden_layers=2, num_attention_heads=2,
           max_position_embeddings=64, cross_attention_frequency=8, spatial_shapes=[2], image_embed_dim=16)


def _stand_ins(monkeypatch, calls):
    """The kernels as torch stand-ins (no rotation, attention = the newest value): each logs (name, positions)."""
    def append(q, k, v, cos, sin, pos, kc, vc, slot):
        calls.append(("rope_qk_append_", q.shape[1]))
        kc[:, slot:slot + q.shape[1]] = k
        vc[:, slot:slot + q.shape[1]] = v

    def append_fp8(q, k, v, cos, sin, pos, k8, v8, ks, vs, slot):
        calls.append(("rope_qk_append_fp8_", q.shape[1]))
        H, s = q.shape[2], int(slot)
        for x, c, sc in ((k, k8, ks), (v, v8, vs)):
            x8, scale = ops.quantize_kv_fp8(x)
            c[:, s:s + q.shape[1]] = x8
            sc[:, s:s + q.shape[1], :H] = scale
            x.copy_((x8.float() * scale[..., None]).to(x.dtype))

    def attention(q, k, v, key_mask=None, causal=True, past=0):
        calls.append(("attention", q.shape[1]))
        return v[:, -q.shape[1]:].reshape(q.shape[0], q.shape[1], -1).contiguous()

    def decode_fp8(q, k8, v8, ks, vs, key_mask=None, causal=True, past=0):
        calls.append(("attention_decode_fp8", q.shape[1]))
        return (v8[:, past].float() * vs[:, past, :q.shape[2], None]).to(q.dtype).reshape(q.shape[0], 1, -1)

    def dequantize(x8, scale, dtype):
        calls.append(("kv_dequantize_fp8", x8.shape[1]))
        return (x8.float() * scale[..., :x8.shape[2], None]).to(dtype)

    for name, fn in (("rope_qk_append_", append), ("rope_qk_append_fp8_", append_fp8), ("attention", attention),
                     ("attention_decode_fp8", decode_fp8), ("kv_dequantize_fp8", dequantize)):
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(ops, "rmsnorm", lambda x, w, eps: (x.float() * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype) * w)
    monkeypatch.setattr(ops, "swiglu", lambda gu: F.silu(gu[..., :gu.shape[-1] // 2]) * gu[..., gu.shape[-1] // 2:])
    monkeypatch.setattr(llama_mmfs.LlamaMMFSAttention, "forward", lambda self, h, *a, **k: h)


def _tiny_model(monkeypatch):
    torch.manual_seed(0)
    m = InterleavedForward(LlamaMMFSConfig(**CFG), orig_vocab_size=38).to(BF16).eval()
    for p in m.parameters():
        p.requires_grad_(False)
    monkeypatch.setattr(m.mm_decoder, "prepare_vision", lambda feats, out=None: PreparedVision(feats.shape))
    return m


def _prompt(B=2, L=6):
    g = torch.Generator().manual_seed(3)
    return generation.Prompt(torch.randn((B, L, CFG["hidden_size"]), generator=g).to(BF16), torch.zeros((B, L, 1)),
                             torch.zeros((B, 1)), torch.ones((B, L), dtype=torch.long),
                             torch.arange(L).repeat(B, 1), [])


def _decode_call(model, p, num_beams, static_cache=True):
    return generation.decode(model, p, 3, 0, static_cache, 0, 1.0, False, 0.9, 1.0, None, num_beams, 1.0, 1)


FP8_OPS = {"rope_qk_append_fp8_", "attention_decode_fp8", "kv_dequantize_fp8"}


@pytest.mark.parametrize("num_beams", [1, 2])
def test_switch_off_never_calls_an_fp8_op(monkeypatch, num_beams):
    calls = []
    _stand_ins(monkeypatch, calls)
    model = _tiny_model(monkeypatch)
    model.enable_fp8_kv_cache().enable_fp8_kv_cache(False)
    _decode_call(model, _prompt(), num_beams)
    assert calls and not FP8_OPS & {c[0] for c in calls}
    assert ("attention", 1) in calls and ("rope_qk_append_", 6) in calls


@pytest.mark.parametrize("num_beams", [1, 2])
def test_switch_on_routes_prefill_and_steps(monkeypatch, num_beams):
    calls, caches = [], []
    _stand_ins(monkeypatch, calls)
    model = _tiny_model(monkeypatch).enable_fp8_kv_cache()
    static_cache = model.mm_decoder.static_cache
    monkeypatch.setattr(model.mm_decoder, "static_cache",
                        lambda *a, **k: caches.append(k.get("kv_fp8")) or static_cache(*a, **k))
    ids = _decode_call(model, _prompt(), num_beams)
    assert ids.shape[0] == 2 and caches and all(caches), "every cache the call allocates is FP8"
    n = CFG["num_hidden_layers"]
    assert calls[:2 * n] == [("rope_qk_append_fp8_", 6), ("attention", 6)] * n     # the prefill from position 0
    steps = calls[2 * n:]
    assert steps and set(steps) == {("rope_qk_append_fp8_", 1), ("attention_decode_fp8", 1)}


def test_prefill_after_cached_positions_dequantises(monkeypatch):
    calls = []
    _stand_ins(monkeypatch, calls)
    model = _tiny_model(monkeypatch)
    cache = model.mm_decoder.static_cache(2, 16, kv_fp8=True)
    assert cache[0].k.dtype == E4M3 and tuple(cache[0].k_scale.shape) == (2, 16, 4)
    x = torch.randn((2, 9, CFG["hidden_size"])).to(BF16)
    with torch.no_grad():
        for a, b in ((0, 4), (4, 8), (8, 9)):
            model.mm_decoder(inputs_embeds=x[:, a:b], past_key_values=cache, use_cache=True)
    n = CFG["num_hidden_layers"]
    assert calls == ([("rope_qk_append_fp8_", 4), ("attention", 4)] * n +
                     [("rope_qk_append_fp8_", 4), ("kv_dequantize_fp8", 8), ("kv_dequantize_fp8", 8), ("attention", 4)] * n +
                     [("rope_qk_append_fp8_", 1), ("attention_decode_fp8", 1)] * n)
    assert cache[0].length == 9


def test_session_and_token_decoder_allocate_fp8_caches(monkeypatch):
    from mm_interleaved_b200.interleaved import InterleavedSession
    model = _tiny_model(monkeypatch)
    for fp8 in (False, True):
        model.enable_fp8_kv_cache(fp8)
        s = InterleavedSession(model, torch.tensor([[1, 5, 6]]), None, torch.zeros((1, 3, 4, 4)), torch.tensor([1]), 12,
                               tokenize_last=False)
        assert all(c.fp8 == fp8 and (c.k.dtype == E4M3) == fp8 for c in s.cache)
        dec = generation.TokenDecoder(model, 2, 256, (2, 1), BF16, "cpu", [2], 0, 0, 4, False)
        assert all(c.fp8 == fp8 for c in dec.past)


def test_cache_row_operations_carry_the_scales():
    H, hd = 2, 16
    src = StaticKV(3, 6, H, hd, BF16, "cpu", kv_fp8=True)
    x8, s = ops.quantize_kv_fp8(torch.randn((3, 6, H, hd)).to(BF16))
    src.k.copy_(x8); src.v.copy_(x8)
    src.k_scale[..., :H] = s; src.v_scale[..., :H] = s
    dst = StaticKV(4, 8, H, hd, BF16, "cpu", kv_fp8=True)
    rows = torch.tensor([2, 0, 0, 1])
    dst.copy_rows_(src, rows, 5)
    assert torch.equal(dst.k[:, :5].view(torch.uint8), x8[rows, :5].view(torch.uint8))
    assert torch.equal(dst.v_scale[:, :5, :H], s[rows, :5])
    dst.reorder_rows_(torch.tensor([3, 3, 1, 0]), 5)
    assert torch.equal(dst.k_scale[:, :5, :H], s[rows[[3, 3, 1, 0]], :5])
    dst.zero_from_(2)
    assert not bool(dst.k[:, 2:].view(torch.uint8).any()) and not bool(dst.v_scale[:, 2:].any())
    with pytest.raises(RuntimeError, match="do not mix"):
        StaticKV(4, 8, H, hd, BF16, "cpu").copy_rows_(src, rows, 5)


def test_static_cache_false_is_refused_while_on(monkeypatch):
    model = _tiny_model(monkeypatch).enable_fp8_kv_cache()
    with pytest.raises(ValueError, match="static_cache=False"):
        _decode_call(model, _prompt(), 1, static_cache=False)


def test_toggling_drops_captured_decode_graphs(monkeypatch):
    model = _tiny_model(monkeypatch).enable_decode_graphs()
    for enabled in (True, False):
        model._decode_graphs["captured"] = object()
        model.enable_fp8_kv_cache(enabled)
        assert model._decode_graphs == {} and model._kv_fp8 == enabled
    assert _tiny_model(monkeypatch).enable_fp8_kv_cache()._decode_graphs is None
    assert not _tiny_model(monkeypatch)._kv_fp8, "off by default"
    off = _tiny_model(monkeypatch).enable_fp8_decode()
    assert not off._kv_fp8, "independent of enable_fp8_decode"
