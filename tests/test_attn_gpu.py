"""GPU parity of the wgmma attention kernel against an fp32 PyTorch statement of
softmax(q k^T / sqrt(d) + mask) v on the same bf16/f16-rounded inputs.

Tolerance, elementwise: P is rounded to the 16-bit type before the second MMA (as in the reference, where
`attn_weights.to(query_states.dtype)` precedes the PV matmul, decoders/modeling_llama_mmfs.py:261-262), so with u the
unit roundoff of the type (2^-9 bf16, 2^-12 f16) every probability carries a relative error <= u and the output one more
rounding:  |err| <= 3 u (P |V|) + u |ref|  (3: rounding of p, ex2.approx, the fp32 row sum and the lazy rescale), evaluated with the
fp32 statement.  Kept beside it: the coarse per-tensor bounds |err| <= 2e-2 max|ref|, mean |err| <= 2e-3 max|ref|."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def eager(q, k, v, km, causal, past, want_bound=False):
    B, Tq, H, hd = q.shape
    Tkv = k.shape[1]
    s = torch.einsum("bqhd,bkhd->bhqk", q.float() * hd ** -0.5, k.float())
    allow = torch.ones((B, 1, Tq, Tkv), dtype=torch.bool, device=q.device)
    if km is not None:
        allow = allow & km[:, None, None, :].bool()
    if causal:
        allow = allow & (torch.arange(Tkv, device=q.device)[None, :] <= past + torch.arange(Tq, device=q.device)[:, None])[None, None]
    s = s.masked_fill(~allow, float("-inf"))
    p = torch.softmax(s, -1).nan_to_num(0.0)
    if want_bound:
        return torch.einsum("bhqk,bkhd->bqhd", p, v.float()), torch.einsum("bhqk,bkhd->bqhd", p, v.float().abs())
    return torch.einsum("bhqk,bkhd->bqhd", p, v.float())


CASES = [
    # B, H, Tq, Tkv, hd, causal, past, masked
    (1, 2, 128, 128, 128, False, 0, False),
    (1, 2, 128, 128, 64, False, 0, False),
    (2, 3, 256, 256, 128, True, 0, False),
    (1, 4, 257, 257, 64, False, 0, False),      # CLIP ViT-L/14: 257 tokens, 16 x 64
    (2, 2, 200, 200, 128, True, 0, True),       # ragged + key padding (left-padded batch)
    (1, 2, 96, 352, 128, True, 256, True),      # chunked prefill on top of a cache
    (1, 5, 512, 512, 128, True, 0, False),      # cfg 2 prefill length
    (1, 2, 1024, 77, 64, False, 0, False),      # SD cross-attention: kv = 77
    (1, 2, 2048, 2048, 128, True, 0, False),    # cfg 3 prefill length
    (2, 2, 640, 640, 128, True, 0, True),       # five query tiles, padding mask
    (1, 3, 1000, 1000, 64, False, 0, False),    # ragged tails of the last query tile and of the key tiles
    (1, 2, 384, 900, 128, True, 516, True),     # chunked prefill on a cache
    (3, 40, 640, 640, 128, True, 0, True),      # 600 items > resident CTAs (1 per SM at hd 128): persistent kernel, masks
    (2, 24, 1000, 1000, 64, False, 0, False),   # persistent, hd 64, ragged tails
    (40, 10, 130, 130, 128, True, 0, False),    # persistent, two-tile items incl. a 2-row query tile
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.timeout(60)
def test_tc_attention_matches_eager(case, dtype):
    from mm_interleaved_b200 import attn_tc, ops
    B, H, Tq, Tkv, hd, causal, past, masked = CASES[case]
    g = torch.Generator().manual_seed(case)
    qkv_q = torch.randn((B, Tq, 3, H, hd), generator=g).to(dtype).to(DEV)       # q is a strided view, like the model's
    q = qkv_q[:, :, 0]
    k = torch.randn((B, Tkv, H, hd), generator=g).to(dtype).to(DEV)
    v = torch.randn((B, Tkv, H, hd), generator=g).to(dtype).to(DEV)
    km = None
    if masked:
        km = torch.ones((B, Tkv), dtype=torch.uint8, device=DEV)
        km[0, :5] = 0
        km[-1, 7:19] = 0
    assert attn_tc.supported(q, k, v, Tq, Tkv, hd)
    out = ops.attention(q, k, v, key_mask=km, causal=causal, past=past).view(B, Tq, H, hd)
    torch.cuda.synchronize()
    ref, pv_abs = eager(q, k, v, km, causal, past, want_bound=True)
    err = (out.float() - ref).abs()
    scale = ref.abs().max()
    assert torch.isfinite(out.float()).all()
    u = 2.0 ** -9 if dtype == torch.bfloat16 else 2.0 ** -12
    bound = 3.0 * u * pv_abs + u * ref.abs() + 1e-6
    assert (err <= bound).all(), float((err / bound).max())
    assert err.max() <= 2e-2 * scale, (err.max().item(), scale.item())
    assert err.mean() <= 2e-3 * scale
    # and the bandwidth kernel agrees on the same problem
    out_g = ops.attention(q, k, v, key_mask=km, causal=causal, past=past, force_generic=True).view(B, Tq, H, hd)
    assert (out_g.float() - ref).abs().max() <= 2e-2 * scale


def test_unsupported_shapes_fall_to_the_bandwidth_kernel_and_errors_are_loud():
    from mm_interleaved_b200 import _lib, attn_tc
    q = torch.randn((1, 64, 2, 80), device=DEV, dtype=torch.bfloat16)
    assert not attn_tc.supported(q, q, q, 64, 64, 80)
    lib = _lib.lib()
    rc = lib.mmfs_attn_forward(q.data_ptr(), q.data_ptr(), q.data_ptr(), q.data_ptr(), None, 1, 2, 64, 64, 80,
                               q.stride(0), q.stride(1), q.stride(0), q.stride(1), q.stride(0), q.stride(1), q.stride(0), q.stride(1),
                               0.1, 0, 0, _lib.BF16, None)
    assert rc == _lib.EUNSUPPORTED


DECODE_CASES = [
    # B, H, Tkv, T_cache, hd, masked
    (3, 5, 700, 1024, 128, True),      # left-padded batch over a pre-allocated cache (views with a larger batch stride)
    (2, 4, 2049, 2049, 128, False),    # cfg-3 decode step
    (1, 3, 1, 8, 64, False),           # first token after a one-token prompt
    (2, 2, 300, 300, 32, False),       # small head
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("case", range(len(DECODE_CASES)))
def test_decode_attention_matches_eager(case, dtype):
    """One query row over a KV cache (split-KV kernel) vs the fp32 eager statement; same tolerances as above, fp32: 1e-5."""
    from mm_interleaved_b200 import ops
    B, H, Tkv, Tc, hd, masked = DECODE_CASES[case]
    g = torch.Generator().manual_seed(100 + case)
    q = torch.randn((B, 1, H, hd), generator=g).to(dtype).to(DEV)
    kc = torch.randn((B, Tc, H, hd), generator=g).to(dtype).to(DEV)
    vc = torch.randn((B, Tc, H, hd), generator=g).to(dtype).to(DEV)
    k, v = kc[:, :Tkv], vc[:, :Tkv]
    km = None
    if masked:
        km = torch.ones((B, Tkv), dtype=torch.uint8, device=DEV)
        km[0, :260] = 0                   # a whole 256-key split is masked
        km[-1, 3:9] = 0
    out = ops.attention(q, k, v, key_mask=km, causal=True, past=Tkv - 1).view(B, 1, H, hd)
    ref = eager(q, k, v, km, True, Tkv - 1)
    scale = ref.abs().max()
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert (out.float() - ref).abs().max() <= tol * scale
    out_g = ops.attention(q, k, v, key_mask=km, causal=True, past=Tkv - 1, force_generic=True).view(B, 1, H, hd)
    assert (out_g.float() - out.float()).abs().max() <= tol * scale
    if masked:                            # a query whose keys are all masked returns zeros (DESIGN.md, attention masks)
        km0 = km.clone(); km0[1] = 0
        z = ops.attention(q, k, v, key_mask=km0, causal=True, past=Tkv - 1).view(B, 1, H, hd)
        assert torch.count_nonzero(z[1]) == 0 and torch.isfinite(z.float()).all()
        # masked cache slots may hold anything (the graphed decoder attends its whole static buffer): NaN there must not leak
        kc2, vc2 = kc.clone(), vc.clone()
        kc2[0, :260] = float("nan"); vc2[0, :260] = float("inf"); kc2[-1, 3:9] = float("nan"); vc2[-1, 3:9] = float("nan")
        o2 = ops.attention(q, kc2[:, :Tkv], vc2[:, :Tkv], key_mask=km, causal=True, past=Tkv - 1).view(B, 1, H, hd)
        assert torch.equal(o2, out)
