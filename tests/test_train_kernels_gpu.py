"""GPU tests of the training-path kernels through the autograd Functions of ``autograd_ops``: each gradient against
float64 autograd of the same op on the same 16-bit inputs, plus the bit-level properties the backward pass relies on
(the forward's output unchanged by the LSE epilogue, fully masked rows with zero gradient, run-to-run identical
results).

Tolerances: u is the unit roundoff of the element type (2^-8 bf16, 2^-11 fp16, an upper bound on the relative error of
one rounding of a normal number; below the smallest normal number the rounding error is absolute, at most u times it).
Row-wise kernels compute in fp32 and round once at the store, so they are held to u * |ref| + u * smallest_normal plus a
few fp32 ulps (2^-16 or tighter) of the magnitude of the terms that cancel in the result, elementwise.  The attention
backward rounds P and dS to 16 bits before its MMAs (as the forward rounds P); those per-entry errors of u average out
over the key / query sums, and the gradients are held to the flash-attention bounds of 1e-2 (bf16) / 2e-3 (fp16) of
max |ref| per tensor -- about 2.5 u and 4 u, since the rounding errors of P, dS and the output add."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
SUB = {t: U[t] * torch.finfo(t).smallest_normal for t in U}     # rounding error of a subnormal result
ATTN_TOL = {torch.bfloat16: 1e-2, torch.float16: 2e-3}
DTYPES = [torch.bfloat16, torch.float16]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _key_mask(B, T, pad):
    """Left padding of ``pad`` keys on the last batch entry (the eval collator's left-padded prompts)."""
    km = torch.ones(B, T, dtype=torch.bool, device="cuda")
    km[-1, :pad] = False
    return km


def _attn_ref(qkv, km, scale):
    """float64 causal attention on (B, T, 3, H, hd): (out (B, T, H, hd), lse (B, H, T)); a row that sees no key has
    output 0, zero gradient and lse +inf."""
    q, k, v = qkv.unbind(2)
    T = q.shape[1]
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    vis = torch.tril(torch.ones(T, T, dtype=torch.bool, device=q.device))[None, None] & km[:, None, None, :]
    seen = vis.any(-1, keepdim=True)
    s = torch.where(seen, torch.where(vis, s, float("-inf")), 0.0)
    p = torch.softmax(s, -1) * seen
    lse = torch.where(seen[..., 0], torch.logsumexp(s, -1), float("inf"))
    return torch.einsum("bhqk,bkhd->bqhd", p, v), lse


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pad", [0, 5])
@pytest.mark.parametrize("T,H", [(16, 2), (200, 3), (1100, 2)])
def test_attention_backward_matches_float64_autograd(T, H, pad, dtype):
    from mm_interleaved_b200 import autograd_ops
    B, hd = 2, 128
    g = _gen(1000 * T + pad)
    qkv = torch.randn(B, T, 3, H, hd, device="cuda", generator=g).to(dtype)
    d_out = torch.randn(B, T, H * hd, device="cuda", generator=g).to(dtype)
    km = _key_mask(B, T, pad)
    scale = hd ** -0.5

    x = qkv.clone().requires_grad_(True)
    autograd_ops.attention(x, km, scale).backward(d_out)
    grad = x.grad.clone()
    x.grad = None
    autograd_ops.attention(x, km, scale).backward(d_out)
    assert torch.equal(grad, x.grad), "two backward runs differ"

    r = qkv.double().requires_grad_(True)
    out_ref, _ = _attn_ref(r, km, scale)
    out_ref.reshape(B, T, H * hd).backward(d_out.double())
    for i, name in enumerate(("dQ", "dK", "dV")):
        ref = r.grad[:, :, i]
        err = (grad[:, :, i].double() - ref).abs().max().item()
        bound = ATTN_TOL[dtype] * ref.abs().max().item()
        assert err <= bound, f"{name}: max err {err:.3e} > {bound:.3e}"
    if pad:   # queries 0..pad-1 of the padded entry see no key; keys 0..pad-1 are seen by none
        assert torch.all(grad[-1, :pad] == 0), "fully masked rows / padded keys must get exactly zero gradient"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("T", [16, 200, 1100])
def test_forward_lse_keeps_the_output_and_matches_logsumexp(T, dtype):
    from mm_interleaved_b200 import ops
    B, H, hd = 2, 3, 128
    qkv = torch.randn(B, T, 3, H, hd, device="cuda", generator=_gen(T)).to(dtype)
    q, k, v = qkv.unbind(2)
    km = _key_mask(B, T, 5)
    with torch.no_grad():
        out, lse = ops.attention_forward_lse(q, k, v, key_mask=km)
        plain = ops.attention(q, k, v, key_mask=km, causal=True).view(B, T, H, hd)
    assert torch.equal(out, plain), "the LSE instantiation must not change O"
    _, lse_ref = _attn_ref(qkv.double(), km, hd ** -0.5)
    finite = torch.isfinite(lse_ref)
    assert torch.all(lse[~finite] == float("inf")) and bool(torch.isfinite(lse[finite]).all())
    # fp32 scores of exact 16-bit products, ex2.approx (2^-22 relative) and an fp32 sum of <= T terms
    err = (lse.double() - lse_ref)[finite].abs()
    assert bool((err <= 1e-5 * lse_ref[finite].abs() + 1e-4).all()), f"lse max err {err.max().item():.3e}"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,cols", [(300, 5120), (2 * 1344 + 7, 1024)])
def test_rmsnorm_backward_matches_float64_autograd(rows, cols, dtype):
    from mm_interleaved_b200 import autograd_ops, ops
    from oracle.mmfs import rms_norm_ref
    eps, u = 1e-6, U[dtype]
    g = _gen(rows + cols)
    x = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    w = (1 + 0.1 * torch.randn(cols, device="cuda", generator=g)).to(dtype)
    dy = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = autograd_ops.rmsnorm(xg, wg, eps)
    with torch.no_grad():
        assert torch.equal(y, ops.rmsnorm(x, w, eps))
    y.backward(dy)

    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    rms_norm_ref(x64, w64, eps).backward(dy.double())
    xd, wd, dyd = x.double(), w.double(), dy.double()
    r = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
    s_abs = (dyd * wd * xd).abs().sum(-1, keepdim=True)
    # dx = r g - x r^3 sum(g x) / N: the two terms cancel, and the fp32 row sum errs by ~2^-19 of sum |g x|
    m = r * (dyd * wd).abs() + xd.abs() * r ** 3 * s_abs / cols
    err = (xg.grad.double() - x64.grad).abs()
    assert bool((err <= u * x64.grad.abs() + 2.0 ** -16 * m + SUB[dtype]).all()), f"dx max err {err.max().item():.3e}"
    # dweight = sum over rows of dy * cast(x r): the cast errs by u/2 per term, the output rounding by u/2
    s_w = (dyd * xd * r).abs().sum(0)
    err = (wg.grad.double() - w64.grad).abs()
    assert bool((err <= u * s_w + u * w64.grad.abs() + SUB[dtype]).all()), f"dweight max err {err.max().item():.3e}"

    with torch.no_grad():
        dx1, dw1 = ops.rmsnorm_backward(x, w, dy, eps)
        dx2, dw2 = ops.rmsnorm_backward(x, w, dy, eps)
        dx3, none = ops.rmsnorm_backward(x, w, dy, eps, weight_grad=False)
    assert torch.equal(dw1, dw2) and torch.equal(dx1, dx2), "the dweight reduction must be bit-reproducible"
    assert torch.equal(dx1, dx3) and none is None and torch.equal(dw1, wg.grad)


@pytest.mark.parametrize("dtype", DTYPES)
def test_swiglu_backward_matches_float64_autograd(dtype):
    from mm_interleaved_b200 import autograd_ops, ops
    rows, inter, u = 96, 1376, U[dtype]
    g = _gen(7)
    gu = (2 * torch.randn(rows, 2 * inter, device="cuda", generator=g)).to(dtype)
    d = torch.randn(rows, inter, device="cuda", generator=g).to(dtype)
    x = gu.clone().requires_grad_(True)
    out = autograd_ops.swiglu(x)
    with torch.no_grad():
        assert torch.equal(out, ops.swiglu(gu))
    out.backward(d)
    r = gu.double().requires_grad_(True)
    gate, up = r.chunk(2, -1)
    (F.silu(gate) * up).backward(d.double())
    gd, ud, dd = gu.double().chunk(2, -1) + (d.double(),)
    # fp32 math, one rounding at the store; silu'(g) = s (1 + g (1 - s)) cancels near g = -1.28
    m = dd.abs() * (ud.abs() * (1 + gd.abs()) + gd.abs())
    err = (x.grad.double() - r.grad).abs()
    assert bool((err <= u * r.grad.abs() + 2.0 ** -18 * torch.cat((m, m), -1) + SUB[dtype]).all()), f"max err {err.max().item():.3e}"


@pytest.mark.parametrize("dtype", DTYPES)
def test_rope_backward_is_the_forward_with_negated_sin(dtype):
    from mm_interleaved_b200 import autograd_ops, ops
    from mm_interleaved_b200.llama_mmfs import rotary_tables
    from oracle.llama import _rotate_half
    B, T, H, hd, u = 2, 50, 3, 128, U[dtype]
    g = _gen(11)
    qkv = torch.randn(B, T, 3, H, hd, device="cuda", generator=g).to(dtype)
    grad = torch.randn(B, T, 3, H, hd, device="cuda", generator=g).to(dtype)
    cos, sin = rotary_tables(hd, 128, device="cuda")
    pos = torch.arange(T, device="cuda").repeat(B, 1)
    pos[1] += 7
    x = qkv.clone().requires_grad_(True)
    y = autograd_ops.rope_qkv(x, cos, sin, pos)
    with torch.no_grad():
        z = qkv.clone()
        ops.rope_qk_(z[:, :, 0], z[:, :, 1], cos, sin, pos)
    assert torch.equal(y, z) and torch.equal(qkv, x.detach()), "out of place, same kernel as the inference path"
    y.backward(grad)
    assert torch.equal(x.grad[:, :, 2], grad[:, :, 2]), "v passes through"

    c, s = cos[pos].double()[:, :, None], sin[pos].double()[:, :, None]     # (B, T, 1, hd)
    r = qkv.double().requires_grad_(True)
    rot = [t * c + _rotate_half(t) * s for t in r[:, :, :2].unbind(2)]
    torch.stack(rot, 2).backward(grad[:, :, :2].double())
    # tables and the two products are each rounded to the element type, then their sum
    gd = grad[:, :, :2].double()
    m = (gd * c[:, :, None]).abs() + _rotate_half((gd * s[:, :, None]).abs()).abs()
    err = (x.grad[:, :, :2].double() - r.grad[:, :, :2]).abs()
    assert bool((err <= u * r.grad[:, :, :2].abs() + 2 * u * m + SUB[dtype]).all()), f"max err {err.max().item():.3e}"


def test_backward_refuses_what_it_does_not_take():
    from mm_interleaved_b200 import autograd_ops
    x = torch.randn(1, 32, 3, 2, 64, device="cuda").to(torch.bfloat16).requires_grad_(True)
    out = autograd_ops.attention(x)                      # the forward takes hd 64 ...
    with pytest.raises(RuntimeError, match="hd = 128"):  # ... the backward does not
        out.sum().backward()
    w = torch.ones(64, device="cuda", requires_grad=True)
    with pytest.raises(RuntimeError, match="bf16"):
        autograd_ops.rmsnorm(torch.randn(4, 64, device="cuda", requires_grad=True), w, 1e-6).sum().backward()
