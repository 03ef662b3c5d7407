"""Decode-step linear (csrc/linear_skinny_sm100.cu) against a plain PyTorch fp32 statement of the same op with the
reference's rounding points (LlamaRMSNorm decoders/modeling_llama_mmfs.py:53-70, LlamaMLP :188-189)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [
    # M, N, K, prologue, residual
    (4, 15360, 5120, 1, False),     # q/k/v of the 13 B decoder with the input RMSNorm folded in
    (4, 5120, 5120, 0, True),       # o_proj + residual (blocks cut by range boundaries: 320 blocks on 132 SMs)
    (4, 27648, 5120, 1, False),     # gate | up with the post-attention RMSNorm
    (4, 5120, 13824, 2, True),      # down_proj of silu(gate) * up, + residual
    (1, 4736, 512, 0, False),       # one step per block
    (8, 1024, 1024, 1, True),       # 8 rows
    (3, 96, 512, 2, False),         # fewer blocks than SMs
    (8, 5120, 5120, 0, True),       # 8 rows at the decoder's width
]


def reference(x, w, res, nw, eps, prologue):
    T = x.dtype
    if prologue == 1:
        xf = x.float()
        xn = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(T)
        a = (nw * xn)
    elif prologue == 2:
        K = x.shape[-1] // 2
        a = torch.nn.functional.silu(x[..., :K].float()).to(T) * x[..., K:]
    else:
        a = x
    y = a.double() @ w.double().t()
    if res is not None:
        y = y + res.double()
    return y, a


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_linear_skinny_matches_fp64_statement(case, dtype):
    from mm_interleaved_b200 import ops
    M, N, K, prologue, with_res = CASES[case]
    g = torch.Generator().manual_seed(500 + case)
    x = torch.randn((M, K * (2 if prologue == 2 else 1)), generator=g).to(dtype).to(DEV)
    w = (torch.randn((N, K), generator=g) * K ** -0.5).to(dtype).to(DEV)
    res = torch.randn((M, N), generator=g).to(dtype).to(DEV) if with_res else None
    nw = (1.0 + 0.1 * torch.randn((K,), generator=g)).to(dtype).to(DEV) if prologue == 1 else None
    assert ops.linear_skinny_supported(x, w, prologue)
    with torch.no_grad():
        y = ops.linear_skinny(x, w, residual=res, norm_weight=nw, eps=1e-6, swiglu=prologue == 2)
        y2 = ops.linear_skinny(x, w, residual=res, norm_weight=nw, eps=1e-6, swiglu=prologue == 2)
        ref, a = reference(x, w, res, nw, 1e-6, prologue)
    assert y.shape == (M, N) and torch.equal(y, y2)                     # timing-independent reduction order
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11          # one rounding of the result ...
    # ... + fp32 accumulation of K exact products (|error| <= K * 2^-24 * sum |a w|, far below) + the operand: when the
    # prologue's fp32 statistics differ in the last bit an element of `a` may round the other way (1 ulp of a, rarely)
    mag = (a.double().abs() @ w.double().abs().t()) + (res.double().abs() if res is not None else 0)
    tol = ulp * ref.abs() + (2.0 ** -22) * mag + (ulp * 4e-3) * mag
    assert ((y.double() - ref).abs() <= tol + 1e-30).all(), float(((y.double() - ref).abs() - tol).max())
    if with_res:                                                         # in place on the residual stream
        buf = res.clone()
        with torch.no_grad():
            out = ops.linear_skinny(x, w, residual=buf, out=buf, norm_weight=nw, eps=1e-6, swiglu=prologue == 2)
        assert out.data_ptr() == buf.data_ptr() and torch.equal(buf, y)


def test_linear_skinny_rejects_what_it_cannot_take():
    from mm_interleaved_b200 import ops
    x = torch.zeros((9, 512), dtype=torch.bfloat16, device=DEV)
    w = torch.zeros((64, 512), dtype=torch.bfloat16, device=DEV)
    assert not ops.linear_skinny_supported(x[:4], torch.zeros((40, 512), dtype=torch.bfloat16, device=DEV))
    assert not ops.linear_skinny_supported(x, w)
    with pytest.raises(RuntimeError):
        ops.linear_skinny(x, w)
    assert not ops.linear_skinny_supported(x[:4], torch.zeros((64, 768), dtype=torch.bfloat16, device=DEV))
    assert not ops.linear_skinny_supported(x[:4].float(), w.float())


def test_decode_step_with_folded_linears_matches_the_cublas_path():
    """A mid-size decoder (hidden 512: the smallest the kernel takes) decoding one token per step over a static cache:
    layers running q/k/v, o_proj, gate/up, down through linear_skinny against the same layers with the kernel disabled
    (cuBLAS + stand-alone RMSNorm / SwiGLU kernels)."""
    from mm_interleaved_b200 import llama_mmfs, ops
    from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, LlamaModel
    cfg = LlamaMMFSConfig(vocab_size=128, hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                          max_position_embeddings=64, cross_attention_frequency=4, spatial_shapes=[4, 2], image_embed_dim=64)
    torch.manual_seed(0)
    model = LlamaModel(cfg).to(DEV, torch.bfloat16).eval()
    B, T = 2, 9
    emb = torch.randn((B, T, 512), device=DEV).to(torch.bfloat16)
    outs = []
    for disabled in (False, True):
        saved = llama_mmfs.SKINNY_DECODE_LINEARS
        llama_mmfs.SKINNY_DECODE_LINEARS = not disabled
        try:
            before = ops.launch_counter[0]
            with torch.no_grad():
                cache = model.static_cache(B, 32)
                o = model(inputs_embeds=emb, past_key_values=cache, use_cache=True, return_dict=True).last_hidden_state[:, -1:]
                steps = [o]
                for _ in range(3):
                    o = model(inputs_embeds=o, past_key_values=cache, use_cache=True, return_dict=True).last_hidden_state
                    steps.append(o)
            outs.append((torch.cat(steps, 1).float(), ops.launch_counter[0] - before))
        finally:
            llama_mmfs.SKINNY_DECODE_LINEARS = saved
    (a, n_a), (b, n_b) = outs
    assert n_a != n_b                                   # the folded path really ran (different kernel count)
    assert (a - b).abs().max() <= 3e-2 * b.abs().max()
