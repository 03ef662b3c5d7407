"""GPU tests of the Q-Former head's training path: the general attention backward and the LayerNorm backward against
float64 autograd, the Q-Former's 16-bit gradients against the reference's own float64 gradients
(tests/golden/qformer_grad_tiny.npz: a fixed sample of each tensor's entries, written by
tests/golden/make_qformer_grad.py), run-to-run identity, the untouched inference path, and
``MMInterleaved.forward(...)["loss"].backward()`` with the tokenizer encoder frozen and its head trainable.

Kernel bounds are those of tests/test_train_kernels_gpu.py: the attention backward rounds P and dS to 16 bits before its
MMAs, so each gradient is held to 1e-2 (bf16) / 2e-3 (fp16) of its max |ref|; the LayerNorm backward computes in fp32
and rounds once, so dx is held to u |ref| plus 2^-16 of the terms that cancel, and dweight / dbias (sums over rows of
fp32 products rounded once) to u |ref| + 2^-16 of the sum of |terms|."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"

from tests.golden.make_golden import tokenizer_state_dict  # noqa: E402
from tests.golden.make_qformer_grad import QFORMER_GRAD_TINY, WEIGHT_SEED, qformer_grad_inputs, sample  # noqa: E402

U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
SUB = {t: U[t] * torch.finfo(t).smallest_normal for t in U}
ATTN_TOL = {torch.bfloat16: 1e-2, torch.float16: 2e-3}
# per-tensor ||g - ref|| / ||ref|| (over the fixture's sample of entries) of the Q-Former's gradients against the reference's float64 ones; both include the
# rounding of the seeded weights and inputs to the element type.  Measured values: DESIGN.md section 4.7.
QFORMER_TOL = {torch.bfloat16: 3e-2, torch.float16: 5e-3}
DTYPES = [torch.bfloat16, torch.float16]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _attn_ref(q, k, v, km, scale):
    """float64 non-causal attention, q (B, Tq, H, hd), k / v (B, Tkv, H, hd); a row that sees no key has output 0."""
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    vis = km[:, None, None, :].expand_as(s)
    seen = vis.any(-1, keepdim=True)
    s = torch.where(seen, torch.where(vis, s, float("-inf")), 0.0)
    p = torch.softmax(s, -1) * seen
    return torch.einsum("bhqk,bkhd->bqhd", p, v)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,Tq,Tkv,masked", [
    (2, 3, 64, 64, False),         # Q-Former self-attention
    (2, 3, 64, 257, False),        # cross-attention to the CLIP tokens
    (2, 3, 50, 131, True),         # ragged tiles and a key-padding mask, one batch entry with every key masked
    (12, 12, 64, 257, True),       # B * H = 144 > the SM count
])
def test_general_attention_backward_matches_float64_autograd(B, H, Tq, Tkv, masked, dtype):
    from mm_interleaved_b200 import autograd_ops, ops
    hd, scale = 64, 64 ** -0.5
    g = _gen(Tq * 1000 + Tkv + B)
    q = torch.randn(B, Tq, H, hd, device=DEV, generator=g).to(dtype)
    kv = torch.randn(B, Tkv, 2, H, hd, device=DEV, generator=g).to(dtype)       # k, v as strided slices of one buffer
    k, v = kv[:, :, 0], kv[:, :, 1]
    d_out = torch.randn(B, Tq, H * hd, device=DEV, generator=g).to(dtype)
    km = torch.ones(B, Tkv, dtype=torch.bool, device=DEV)
    if masked:
        km[0, Tkv // 3:] = False
        km[-1] = False

    xs = [t.clone().requires_grad_(True) for t in (q, k, v)]
    out = autograd_ops.attention_general(*xs, key_mask=km if masked else None, scale=scale)
    if Tq >= 16:
        with torch.no_grad():
            plain = ops.attention(q, k, v, key_mask=km if masked else None, causal=False)
        assert torch.equal(out, plain), "the LSE forward must give the inference kernel's output"
    out.backward(d_out)
    grads = [x.grad.clone() for x in xs]
    for x in xs:
        x.grad = None
    autograd_ops.attention_general(*xs, key_mask=km if masked else None, scale=scale).backward(d_out)
    for a, x in zip(grads, xs):
        assert torch.equal(a, x.grad), "two backward runs differ"

    rs = [t.double().requires_grad_(True) for t in (q, k, v)]
    _attn_ref(*rs, km, scale).reshape(B, Tq, H * hd).backward(d_out.double())
    for name, got, r in zip(("dQ", "dK", "dV"), grads, rs):
        err = (got.double() - r.grad).abs().max().item()
        bound = ATTN_TOL[dtype] * r.grad.abs().max().item()
        assert err <= bound, f"{name}: max err {err:.3e} > {bound:.3e}"
    if masked:
        assert torch.all(grads[0][-1] == 0) and torch.all(grads[1][-1] == 0) and torch.all(grads[2][-1] == 0)
        assert torch.all(grads[1][0, Tkv // 3:] == 0) and torch.all(grads[2][0, Tkv // 3:] == 0)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,cols", [(12 * 257 * 2 + 5, 64), (2 * 64 + 3, 768), (2 * 257, 1024), (300, 8192)])
def test_layernorm_backward_matches_float64_autograd(rows, cols, dtype):
    from mm_interleaved_b200 import autograd_ops, ops
    eps, u = 1e-6, U[dtype]
    g = _gen(rows + cols)
    x = (0.5 + torch.randn(rows, cols, device=DEV, generator=g)).to(dtype)
    w = (1 + 0.1 * torch.randn(cols, device=DEV, generator=g)).to(dtype)
    b = (0.1 * torch.randn(cols, device=DEV, generator=g)).to(dtype)
    dy = torch.randn(rows, cols, device=DEV, generator=g).to(dtype)
    xg, wg, bg = (t.clone().requires_grad_(True) for t in (x, w, b))
    y = autograd_ops.layernorm(xg, wg, bg, eps)
    with torch.no_grad():
        assert torch.equal(y, ops.layernorm(x, w, b, eps))
    y.backward(dy)

    x64, w64, b64 = (t.double().requires_grad_(True) for t in (x, w, b))
    F.layer_norm(x64, (cols,), w64, b64, eps).backward(dy.double())
    xd, wd, dyd = x.double(), w.double(), dy.double()
    r = torch.rsqrt(xd.var(-1, unbiased=False, keepdim=True) + eps)
    xh = (xd - xd.mean(-1, keepdim=True)) * r
    gg = (dyd * wd).abs()
    # dx = r (g - mean(g) - xhat mean(g xhat)): the three terms cancel; fp32 sums err by ~2^-19 of their |terms|
    m = r * (gg + gg.mean(-1, keepdim=True) + xh.abs() * (gg * xh.abs()).mean(-1, keepdim=True))
    err = (xg.grad.double() - x64.grad).abs()
    assert bool((err <= u * x64.grad.abs() + 2.0 ** -16 * m + SUB[dtype]).all()), f"dx max err {err.max().item():.3e}"
    for name, got, ref, s in (("dweight", wg.grad, w64.grad, (dyd * xh).abs().sum(0)), ("dbias", bg.grad, b64.grad, dyd.abs().sum(0))):
        err = (got.double() - ref).abs()
        assert bool((err <= u * ref.abs() + 2.0 ** -16 * s + SUB[dtype]).all()), f"{name} max err {err.max().item():.3e}"

    with torch.no_grad():
        a = ops.layernorm_backward(x, w, dy, eps)
        c = ops.layernorm_backward(x, w, dy, eps)
        dx_only = ops.layernorm_backward(x, w, dy, eps, weight_grad=False, bias_grad=False)
    assert all(torch.equal(p, q) for p, q in zip(a, c)), "the dweight / dbias reduction must be bit-reproducible"
    assert torch.equal(a[0], dx_only[0]) and dx_only[1] is None and dx_only[2] is None
    assert torch.equal(a[1], wg.grad) and torch.equal(a[2], bg.grad)


def _qformer(dtype):
    from mm_interleaved_b200 import visual_tokenizer as vt
    per = vt.PerceiverResampler(**QFORMER_GRAD_TINY)
    sd = tokenizer_state_dict(per.state_dict(), seed=WEIGHT_SEED)
    z = np.load(os.path.join(GOLDEN, "qformer_grad_tiny.npz"))
    assert sorted(sd.keys()) == [str(k) for k in z["keys"]]
    chk = float(sum(v.double().sum() for v in sd.values()))
    assert abs(chk - float(z["checksum"])) <= 1e-6 * max(1.0, abs(chk))
    per.load_state_dict(sd, strict=True)
    return per.to(DEV, dtype).train(), z


def _qformer_grads(per, dtype, masked):
    enc, mask, proj = qformer_grad_inputs()
    per.zero_grad(set_to_none=True)
    e = enc.to(DEV, dtype).requires_grad_(True)
    out = per(encoder_hidden_states=e, encoder_attention_mask=mask.to(DEV) if masked else None)[0]
    (out.double() * proj.to(DEV)).sum().backward()
    grads = {n: p.grad.clone() for n, p in per.named_parameters()}
    grads["encoder_hidden_states"] = e.grad.clone()
    return out.detach(), grads


@pytest.mark.parametrize("dtype", DTYPES)
def test_qformer_gradients_match_reference_golden(dtype):
    torch.backends.cuda.matmul.allow_tf32 = False
    per, z = _qformer(dtype)
    worst = {}
    for tag in ("masked", "unmasked"):
        out, grads = _qformer_grads(per, dtype, tag == "masked")
        want = torch.from_numpy(z[f"{tag}/out"]).double()
        assert float((sample(out.double().cpu()) - want).norm() / want.norm()) <= QFORMER_TOL[dtype]
        assert set(grads) == {k.split("/", 1)[1] for k in z.files if k.startswith(tag + "/")} - {"out"}
        rel = {}
        for n, g in grads.items():
            ref = torch.from_numpy(z[f"{tag}/{n}"]).double()
            # a shift of every key by the k_norm bias shifts a query's scores by one constant, which the softmax removes:
            # that gradient is exactly 0 and the reference's is float64 round-off, so the error is measured against the
            # scale of the sibling k_norm.weight gradient instead
            scale = torch.from_numpy(z[f"{tag}/{n[:-4]}weight"]).norm() if n.endswith("k_norm.bias") else ref.norm()
            rel[n] = float((sample(g.double().cpu()) - ref).norm()) / max(float(scale), 1e-30)
        worst[tag] = {n: f"{e:.1e}" for n, e in sorted(rel.items(), key=lambda t: -t[1])[:3]}
        bad = {n: f"{e:.2e}" for n, e in rel.items() if e > QFORMER_TOL[dtype]}
        print(f"qformer grads {dtype} {tag}: largest per-tensor relative errors {worst[tag]}")
        assert not bad, f"{tag}: relative errors above {QFORMER_TOL[dtype]}: {bad}"


def test_qformer_backward_is_run_to_run_identical():
    per, _ = _qformer(torch.bfloat16)
    _, a = _qformer_grads(per, torch.bfloat16, True)
    _, b = _qformer_grads(per, torch.bfloat16, True)
    for n in a:
        assert torch.equal(a[n], b[n]), n


def test_tokenizer_inference_output_is_untouched_by_trainable_head():
    """Under torch.no_grad() a tokenizer whose head requires grad runs the inference path: bit-identical outputs."""
    from tests.test_mm_interleaved_gpu import _batch, _build
    model, _ = _build()
    tok = model.visual_tokenizer.to(torch.bfloat16)
    images = _batch()[1].to(DEV, torch.bfloat16)
    tok.requires_grad_(False)
    with torch.no_grad():
        ref = tok(images)
    tok.requires_grad_(True)
    tok.encoder.requires_grad_(False)
    with torch.no_grad():
        got = tok(images)
    assert torch.equal(got["vis_embed"], ref["vis_embed"]) and torch.equal(got["image_embeds"], ref["image_embeds"])
    for a, b in zip(got["multiscale_features"], ref["multiscale_features"]):
        assert torch.equal(a, b)


def test_mm_interleaved_loss_backward_trains_the_tokenizer_head():
    """Encoder frozen, head trainable (Q-Former at head dim 64): ``forward(...)["loss"].backward()`` equals the same loss
    spelled out at module level, gradient for gradient; a trainable encoder still raises."""
    from tests.test_mm_interleaved_gpu import _batch, _build
    model, _ = _build()
    model = model.to(torch.bfloat16).freeze_like_reference()
    ids, images, nimg, mask = _batch()
    batch = dict(text_ids=ids.to(DEV), image_tensors=images.to(DEV), num_image_per_seq=nimg.to(DEV),
                 attention_mask=mask.to(DEV), meta={"dataset_name": "synthetic"})
    with pytest.raises(RuntimeError, match="the visual tokenizer has no backward"):
        model(**batch)
    model.visual_tokenizer.encoder.requires_grad_(False)

    model(**batch)["loss"].backward()
    trainable = [(n, p) for n, p in model.named_parameters()
                 if p.requires_grad and n.split(".")[0] in ("mm_decoder", "text_decoder", "soi_token", "visual_tokenizer")]
    names = {n for n, _ in trainable}
    head = {n for n in names if n.startswith("visual_tokenizer.")}
    for part in ("pos_proj.weight", "pos_ln.weight", "post_ln.bias", "proj.weight", "perceiver_resampler.queries",
                 "blip2qformer.encoder.layer.0.crossattention.attention.k_norm.weight",
                 "blip2qformer.encoder.layer.1.attention.attention.query.weight"):
        assert any(n.endswith(part) for n in head), part
    got = {n: p.grad.clone() for n, p in trainable}
    assert all(g is not None and bool(torch.isfinite(g).all()) for g in got.values())
    assert all(float(got[n].abs().max()) > 0 for n in head), "a head tensor got no gradient"
    model.zero_grad(set_to_none=True)

    n_img = batch["num_image_per_seq"].reshape(-1)
    vis = model.visual_tokenizer(batch["image_tensors"].to(torch.bfloat16))
    mm_embeds, cross, feats = model.prepare(batch["text_ids"], vis, n_img, int(n_img.max()))
    hidden = model.mm_decoder(inputs_embeds=mm_embeds, attention_mask=batch["attention_mask"], vision_hidden_states=feats,
                              cross_attention_mask=cross, use_cache=False).last_hidden_state
    logits = model.text_decoder.logits(hidden)
    gt = model._prepare_gt_text_ids(batch["text_ids"], batch["attention_mask"], 0, None, batch["meta"])
    F.cross_entropy(logits[:, :-1].float().transpose(1, 2), gt.contiguous()).backward()
    for n, p in trainable:
        assert torch.equal(p.grad, got[n]), n
