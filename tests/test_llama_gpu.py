"""GPU parity of the H100 Llama-MMFS decoder and its kernels.

Tolerances: fp32 model output vs the reference's fp32 golden: |err| <= 1e-3*|ref| + 2e-5 at non-padding
positions (north-star 1e-3 rel; fully masked = padding query rows are unspecified, DESIGN.md);
kernels in fp32 vs a plain PyTorch fp32 statement of the same op: 1e-5 / 1e-4; bf16 kernels: one bf16 ulp.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import error_metrics  # noqa: E402
from oracle.llama import additive_mask_ref, rotary_tables_ref  # noqa: E402
from oracle.mmfs import rms_norm_ref  # noqa: E402
from tests.golden.make_golden import LLAMA_TC, LLAMA_TINY, llama_inputs, seeded_state_dict  # noqa: E402
from tests.test_oracle_llama import tiny_state_dict  # noqa: E402

DEV = "cuda"


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_rmsnorm_matches_reference_formula(dtype):
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn((3, 7, 5120), generator=g).to(dtype)
    w = (1 + 0.1 * torch.randn(5120, generator=g)).to(dtype)
    y = ops.rmsnorm(x.to(DEV), w.to(DEV), 1e-6).cpu()
    ref = rms_norm_ref(x, w, 1e-6)
    if dtype == torch.float32:
        assert (y - ref).abs().max() < 1e-5
    else:
        assert ((y.float() - ref.float()).abs() <= ref.float().abs() * 2 ** -7 + 1e-6).all()
        assert (y == ref).float().mean() > 0.98


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_rope_matches_reference_formula(dtype):
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(1)
    B, T, H, hd = 2, 9, 3, 128
    qkv = torch.randn((B, T, 3, H, hd), generator=g).to(dtype)
    pos = torch.stack([torch.arange(T), (torch.arange(T) - 2).clamp(min=0)])
    cos, sin = rotary_tables_ref(hd, 64)
    d = qkv.to(DEV).clone()
    ops.rope_qk_(d[:, :, 0], d[:, :, 1], cos.to(DEV), sin.to(DEV), pos.to(DEV))
    c = cos.to(dtype)[pos][:, :, None]
    s = sin.to(dtype)[pos][:, :, None]
    rot = lambda x: torch.cat((-x[..., hd // 2:], x[..., : hd // 2]), -1)
    for i in (0, 1):
        ref = qkv[:, :, i] * c + rot(qkv[:, :, i]) * s
        got = d[:, :, i].cpu()
        if dtype == torch.float32:
            assert (got - ref).abs().max() < 1e-6
        else:
            assert ((got.float() - ref.float()).abs() <= ref.float().abs() * 2 ** -7 + 1e-3).all()
    assert torch.equal(d[:, :, 2].cpu(), qkv[:, :, 2])    # v untouched


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("device_slot", [False, True])
def test_rope_append_equals_rope_then_copy(dtype, device_slot):
    """The fused RoPE + KV-cache append writes bit-for-bit what rope_qk_ followed by the two cache copies wrote."""
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(3)
    B, T, H, hd, Tmax, slot = 2, (1 if device_slot else 7), 3, 128, 20, 5
    qkv = torch.randn((B, T, 3, H, hd), generator=g).to(dtype).to(DEV)
    pos = (torch.arange(T)[None] + torch.tensor([[slot], [slot - 2]])).to(DEV)
    cos, sin = (t.to(DEV) for t in rotary_tables_ref(hd, 64))
    ref = qkv.clone()
    ops.rope_qk_(ref[:, :, 0], ref[:, :, 1], cos, sin, pos)
    kc = torch.full((B + 1, Tmax, H, hd), 7.0, dtype=dtype, device=DEV)[:B]      # a view with a larger batch extent
    vc = torch.full((B + 1, Tmax, H, hd), 7.0, dtype=dtype, device=DEV)[:B]
    got = qkv.clone()
    ops.rope_qk_append_(got[:, :, 0], got[:, :, 1], got[:, :, 2], cos, sin, pos, kc, vc,
                        torch.tensor([slot], device=DEV) if device_slot else slot)
    assert torch.equal(got[:, :, 0], ref[:, :, 0])                                  # q rotated in place
    assert torch.equal(got[:, :, 1], qkv[:, :, 1]) and torch.equal(got[:, :, 2], qkv[:, :, 2])   # k, v operands untouched
    assert torch.equal(kc[:, slot:slot + T], ref[:, :, 1]) and torch.equal(vc[:, slot:slot + T], qkv[:, :, 2])
    for c in (kc, vc):                                                              # nothing else written
        assert (c[:, :slot] == 7).all() and (c[:, slot + T:] == 7).all()
    if not device_slot:
        with pytest.raises(RuntimeError):
            ops.rope_qk_append_(got[:, :, 0], got[:, :, 1], got[:, :, 2], cos, sin, pos, kc, vc, Tmax - T + 1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_swiglu_matches_reference_formula(dtype):
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(2)
    gu = torch.randn((5, 3, 2 * 512), generator=g).to(dtype)
    y = ops.swiglu(gu.to(DEV)).cpu()
    ref = torch.nn.functional.silu(gu[..., :512]) * gu[..., 512:]
    tol = 1e-6 if dtype == torch.float32 else 2 ** -7
    assert ((y.float() - ref.float()).abs() <= ref.float().abs() * tol + 1e-6).all()


@pytest.mark.parametrize("shape", [(2, 3, 17, 17, 128, 0), (1, 2, 1, 40, 128, 39), (2, 4, 33, 33, 64, 0), (1, 2, 5, 300, 80, 295)])
@pytest.mark.parametrize("causal", [True, False])
def test_generic_attention_matches_eager(shape, causal):
    from mm_interleaved_b200 import ops
    B, H, Tq, Tkv, hd, past = shape
    g = torch.Generator().manual_seed(3)
    q = torch.randn((B, Tq, H, hd), generator=g)
    k = torch.randn((B, Tkv, H, hd), generator=g)
    v = torch.randn((B, Tkv, H, hd), generator=g)
    km = torch.ones((B, Tkv), dtype=torch.bool)
    km[0, :3] = False
    out = ops.attention(q.to(DEV), k.to(DEV), v.to(DEV), key_mask=km.to(DEV), causal=causal, past=past,
                        force_generic=True).cpu().view(B, Tq, H, hd)
    s = torch.einsum("bqhd,bkhd->bhqk", q * hd ** -0.5, k)
    allow = km[:, None, None, :].expand(B, H, Tq, Tkv).clone()
    if causal:
        allow &= (torch.arange(Tkv)[None, :] <= past + torch.arange(Tq)[:, None])[None, None]
    s = s.masked_fill(~allow, float("-inf"))
    p = torch.softmax(s, -1).nan_to_num(0.0)
    ref = torch.einsum("bhqk,bkhd->bqhd", p, v)
    assert (out - ref).abs().max() < 2e-5


def build_model(dtype):
    model, sd, z = tiny_state_dict()
    model.load_state_dict(sd, strict=True)
    return model.to(DEV, dtype).eval(), z


def test_model_fp32_prefill_and_decode_match_reference_golden():
    model, z = build_model(torch.float32)
    embeds, vision, attn_mask, position_ids, cross = llama_inputs(LLAMA_TINY, 2, 12, 2, seed=99)
    with torch.no_grad():
        out = model(inputs_embeds=embeds.to(DEV), attention_mask=attn_mask.to(DEV), position_ids=position_ids.to(DEV),
                    vision_hidden_states=vision.to(DEV), cross_attention_mask=cross.to(DEV), use_cache=True)
        ref = torch.from_numpy(z["prefill_fp32"])
        valid = attn_mask.bool()
        err = (out.last_hidden_state.cpu() - ref).abs()[valid]
        assert (err <= 1e-3 * ref[valid].abs() + 2e-5).all(), err.max()
        g = torch.Generator().manual_seed(7)
        step = torch.randn((2, 1, LLAMA_TINY["hidden_size"]), generator=g)
        attn2 = torch.cat([attn_mask, torch.ones((2, 1), dtype=torch.long)], 1)
        cross2 = torch.cat([cross, cross[:, -1:]], 1)
        out2 = model(inputs_embeds=step.to(DEV), attention_mask=attn2.to(DEV), position_ids=(position_ids[:, -1:] + 1).to(DEV),
                     past_key_values=out.past_key_values, vision_hidden_states=vision.to(DEV),
                     cross_attention_mask=cross2.to(DEV), use_cache=True)
        ref2 = torch.from_numpy(z["decode_fp32"])
        err2 = (out2.last_hidden_state.cpu() - ref2).abs()
        assert (err2 <= 1e-3 * ref2.abs() + 2e-5).all(), err2.max()
        assert out2.past_key_values[0][0].shape[1] == 13


def test_model_bf16_tracks_fp32_reference():
    model, z = build_model(torch.bfloat16)
    embeds, vision, attn_mask, position_ids, cross = llama_inputs(LLAMA_TINY, 2, 12, 2, seed=99)
    with torch.no_grad():
        out = model(inputs_embeds=embeds.to(DEV, torch.bfloat16), attention_mask=attn_mask.to(DEV),
                    position_ids=position_ids.to(DEV), vision_hidden_states=vision.to(DEV, torch.bfloat16),
                    cross_attention_mask=cross.to(DEV), use_cache=False)
    ref = torch.from_numpy(z["prefill_fp32"])
    valid = attn_mask.bool()
    err = (out.last_hidden_state.float().cpu() - ref).abs()[valid]
    assert err.max() <= 6e-2 * ref[valid].abs().max()      # bf16 storage through 3 layers


@pytest.mark.parametrize("dtype,max_tol,rms_tol", [(torch.float16, 3.0e-3, 2.5e-3), (torch.bfloat16, 2.5e-2, 2.0e-2),
                                                   (torch.float32, 1.0e-5, 1.0e-5)])
def test_long_prompt_takes_the_tcgen05_kernel_and_tracks_the_reference_golden(dtype, max_tol, rms_tol):
    """A 200-token left-padded prompt through the tiny decoder in 16 bit: every layer's self-attention goes through the
    wgmma kernel (two query tiles, four key tiles, padding mask, causal diagonal) and every second layer through the
    fused MMFS sampler -- jointly against the fp32 output of the REFERENCE LlamaModel on the same weights and inputs
    (tests/golden/llama_tc.npz, generated by make_golden.make_llama_tc from the reference's own modeling file).
    Tolerances are for 16-bit storage through 3 layers: max error relative to max |ref|, and relative RMS error.  fp32
    takes the bandwidth kernel (the tensor-core kernel is 16-bit only) and must match to 1e-5."""
    import os

    import numpy as np
    from mm_interleaved_b200 import attn_tc
    from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, LlamaModel
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "llama_tc.npz"))
    model = LlamaModel(LlamaMMFSConfig(**{**LLAMA_TINY, "max_position_embeddings": 256}))
    sd = seeded_state_dict(model.state_dict(), seed=4242)
    assert abs(float(sum(v.double().sum() for v in sd.values())) - float(z["weight_checksum"])) < 1e-6
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV, dtype).eval()
    c = LLAMA_TC
    embeds, vision, attn_mask, position_ids, cross = llama_inputs(LLAMA_TINY, c["B"], c["T"], c["n_img"], seed=c["seed"], left_pad=c["left_pad"])
    calls, real = [], attn_tc.forward

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)

    attn_tc.forward = spy
    try:
        with torch.no_grad():
            out = model(inputs_embeds=embeds.to(DEV, dtype), attention_mask=attn_mask.to(DEV), position_ids=position_ids.to(DEV),
                        vision_hidden_states=vision.to(DEV, dtype), cross_attention_mask=cross.to(DEV), use_cache=False)
    finally:
        attn_tc.forward = real
    assert len(calls) == (0 if dtype == torch.float32 else LLAMA_TINY["num_hidden_layers"])   # tensor-core kernel in every layer
    ref = torch.from_numpy(z["prefill_fp32"])
    valid = attn_mask.bool()
    got = out.last_hidden_state.float().cpu()
    err = (got - ref)[valid]
    assert torch.isfinite(got[valid]).all()
    assert err.abs().max() <= max_tol * ref[valid].abs().max(), float(err.abs().max() / ref[valid].abs().max())
    assert err.pow(2).mean().sqrt() <= rms_tol * ref[valid].pow(2).mean().sqrt(), float(err.pow(2).mean().sqrt() / ref[valid].pow(2).mean().sqrt())


FULL_WIDTH = dict(vocab_size=64, hidden_size=5120, intermediate_size=13824, num_hidden_layers=2, num_attention_heads=40,
                  max_position_embeddings=2048, rms_norm_eps=1e-6, pad_token_id=0, cross_attention_frequency=2,
                  spatial_shapes=[32, 16, 8], image_embed_dim=1024)


@pytest.mark.parametrize("dtype,max_tol,rms_tol", [(torch.float32, 2e-4, 2e-5), (torch.bfloat16, 4e-2, 1.5e-2)])
def test_full_width_layers_match_the_oracle(dtype, max_tol, rms_tol):
    """Two decoder layers at the 13 B model's REAL widths (hidden 5120, 40 heads of 128, MLP 13824, MMFS with 16 heads x 64
    over 32^2 + 16^2 + 8^2 feature maps of 3 images, seeded weights): one MMFS layer + one plain layer on a 160-token
    left-padded prompt against the oracle restatement of the reference layers (oracle/llama.py, pinned by the tiny
    goldens) on the host.  fp32 takes the bandwidth attention kernel and the generic sampler's fp32 path; bf16 the
    wgmma kernel and the specialised 16-bit sampler -- the kernels and shapes of the benchmarked step."""
    from oracle.llama import llama_model_ref
    from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, LlamaModel
    model = LlamaModel(LlamaMMFSConfig(**FULL_WIDTH))
    sd = seeded_state_dict(model.state_dict(), seed=777)
    model.load_state_dict(sd, strict=True)
    B, T, n_img = 2, 160, 3
    embeds, vision, attn_mask, position_ids, cross = llama_inputs(FULL_WIDTH, B, T, n_img, seed=5, left_pad=7)
    cfg = dict(eps=1e-6, n_heads=40, n_layers=2, spatial_shapes=[(s, s) for s in FULL_WIDTH["spatial_shapes"]])
    ref, _ = llama_model_ref(sd, embeds, attn_mask, position_ids, vision, cross, cfg)
    model = model.to(DEV, dtype).eval()
    with torch.no_grad():
        out = model(inputs_embeds=embeds.to(DEV, dtype), attention_mask=attn_mask.to(DEV), position_ids=position_ids.to(DEV),
                    vision_hidden_states=vision.to(DEV, dtype), cross_attention_mask=cross.to(DEV), use_cache=False)
    valid = attn_mask.bool()
    got = out.last_hidden_state.float().cpu()
    err = (got - ref)[valid]
    assert torch.isfinite(got[valid]).all()
    assert err.abs().max() <= max_tol * ref[valid].abs().max(), float(err.abs().max() / ref[valid].abs().max())
    assert err.pow(2).mean().sqrt() <= rms_tol * ref[valid].pow(2).mean().sqrt(), float(err.pow(2).mean().sqrt() / ref[valid].pow(2).mean().sqrt())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("cols", [64, 320, 768, 1024, 1280, 2048, 5120, 100])
def test_layernorm_matches_torch(cols, dtype):
    """Warp-per-row path (cols <= 2048 bf16 / 1024 fp32, 16-byte aligned) and the block fallback (5120, 100)."""
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(cols)
    x = (torch.randn((3, 37, cols), generator=g) * 2 + 0.5).to(dtype)
    w = (1 + 0.1 * torch.randn(cols, generator=g)).to(dtype)
    b = (0.1 * torch.randn(cols, generator=g)).to(dtype)
    y = ops.layernorm(x.to(DEV), w.to(DEV), b.to(DEV), 1e-6).float().cpu()
    ref = torch.nn.functional.layer_norm(x.float(), (cols,), w.float(), b.float(), 1e-6)
    tol = 2e-5 if dtype == torch.float32 else 2e-2
    assert (y - ref).abs().max() <= tol
    y2 = ops.layernorm(x.to(DEV), None, None, 1e-6).float().cpu()
    assert (y2 - torch.nn.functional.layer_norm(x.float(), (cols,), None, None, 1e-6)).abs().max() <= tol
