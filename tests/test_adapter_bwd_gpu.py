"""GPU tests of the ViT-Adapter's training path: the quick-GELU and bilinear-resize backward kernels, the CLIP
self-attention backward into one QKV gradient and the MSDA backward at the adapter's shapes against float64 autograd; the
whole tokenizer's 16-bit gradients against the reference's own float64 ones (tests/golden/adapter_grad_tiny.npz, written
by tests/golden/make_adapter_grad.py); bit-identical outputs under autograd, run-to-run identical gradients, and
``MMInterleaved.forward(...)["loss"].backward()`` with the adapter and head trainable.

Bounds: the quick-GELU and resize backward compute in fp32 and round once, so each element is held to u |ref| plus
2^-20 of the sum of the magnitudes of its terms (fp32 rounding of terms that cancel) plus a subnormal floor; attention
and MSDA use the bounds of tests/test_qformer_bwd_gpu.py and tests/test_msda_bwd_gpu.py.  The SPM, DWConv and
``adapter_up`` gradients come from cuDNN, which is run-to-run identical only with ``cudnn.deterministic`` (a fixture
here sets it and restores it)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"

from oracle import make_msda_inputs, msda_core_pytorch  # noqa: E402
from tests.golden.make_adapter_grad import ADAPTER_GRAD_TINY, OUTPUTS, WEIGHT_SEED, adapter_grad_inputs, flat_outputs  # noqa: E402
from tests.golden.make_golden import tokenizer_state_dict  # noqa: E402
from tests.golden.make_qformer_grad import sample  # noqa: E402

U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
SUB = {t: U[t] * torch.finfo(t).smallest_normal for t in U}
ATTN_TOL = {torch.bfloat16: 1e-2, torch.float16: 2e-3}
# per-tensor ||g - ref|| / ||ref|| over the fixture's sample, against the reference's float64 gradients (both include the
# rounding of the seeded weights and inputs to the element type), by class (_grad_class): "location", the consumers of
# the MSDA location gradient, which is discontinuous at pixel boundaries that 16-bit sampling locations move points
# across; "pool", the SPM stem in front of the max-pool, whose 16-bit forward routes some windows' gradient to another
# pixel (test_spm_backward_per_stage); "rest", every other tensor.  Measured values and analysis: DESIGN.md section 6.
# The median of "rest" is held to the Q-Former's bounds (QFORMER_TOL).
ADAPTER_TOL = {"location": {torch.bfloat16: 0.6, torch.float16: 0.1},
               "pool": {torch.bfloat16: 0.3, torch.float16: 0.15},
               "rest": {torch.bfloat16: 0.2, torch.float16: 2e-2}}
QFORMER_TOL = {torch.bfloat16: 3e-2, torch.float16: 5e-3}
DTYPES = [torch.bfloat16, torch.float16]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.fixture
def deterministic_cudnn():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(4 * 257, 4096), (3 * 257 + 1, 1027)])      # CLIP MLP; a ragged scalar tail
def test_quick_gelu_backward_matches_float64_autograd(shape, dtype):
    from mm_interleaved_b200 import autograd_ops, ops
    g = _gen(shape[1])
    h = (2.5 * torch.randn(shape, device=DEV, generator=g)).to(dtype)
    dy = torch.randn(shape, device=DEV, generator=g).to(dtype)
    hg = h.clone().requires_grad_(True)
    y = autograd_ops.quick_gelu(hg)
    assert torch.equal(y, h * torch.sigmoid(1.702 * h)), "the Function's forward must give the inference bits"
    y.backward(dy)
    with torch.no_grad():
        assert torch.equal(ops.quick_gelu_backward(h, dy), hg.grad)
    h64 = h.double().requires_grad_(True)
    (h64 * torch.sigmoid(1.702 * h64)).backward(dy.double())
    hd, dyd = h.double(), dy.double()
    s = torch.sigmoid(1.702 * hd)
    terms = dyd.abs() * (s + (1.702 * hd * s * (1 - s)).abs())
    err = (hg.grad.double() - h64.grad).abs()
    bound = U[dtype] * h64.grad.abs() + 2.0 ** -20 * terms + SUB[dtype]
    assert bool((err <= bound).all()), f"max err {err.max().item():.3e}, worst ratio {(err / bound).max().item():.3f}"


def _resize_dy(B, C, Ho, Wo, layout, dtype, g):
    if layout == "nchw":
        return torch.randn(B, C, Ho, Wo, device=DEV, generator=g).to(dtype)
    # the gradient pack_mmfs_features' backward hands over: (B, Ho*Wo, C) tokens viewed as NCHW
    return torch.randn(B, Ho * Wo, C, device=DEV, generator=g).to(dtype).transpose(1, 2).reshape(B, C, Ho, Wo)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layout", ["nchw", "tokens"])
@pytest.mark.parametrize("side", [16, 8, 4, 2])              # 2: x0.5 gives a 1 x 1 map (size-1 dims, any strides)
@pytest.mark.parametrize("factor", [4, 2, 0.5])
def test_resize_bilinear_backward_matches_float64_autograd(factor, side, layout, dtype):
    from mm_interleaved_b200 import autograd_ops
    B, C = 3, 136
    g = _gen(side * 10 + int(factor * 2))
    x_tok = torch.randn(B, side * side, C, device=DEV, generator=g).to(dtype)
    Ho = int(side * factor)
    dy = _resize_dy(B, C, Ho, Ho, layout, dtype, g)
    grads = []
    for _ in range(2):
        xt = x_tok.clone().requires_grad_(True)
        x = xt.transpose(1, 2).reshape(B, C, side, side)                    # the adapter's stage-output view
        y = autograd_ops.resize_bilinear(x, factor)
        with torch.no_grad():
            assert torch.equal(y, F.interpolate(x, scale_factor=factor, mode="bilinear", align_corners=False))
        y.backward(dy)
        grads.append(xt.grad)
    assert torch.equal(grads[0], grads[1]), "two backward runs differ"
    x64 = x_tok.double().transpose(1, 2).reshape(B, C, side, side).requires_grad_(True)
    F.interpolate(x64, scale_factor=factor, mode="bilinear", align_corners=False).backward(dy.double())
    want = x64.grad.flatten(2).transpose(1, 2)
    a64 = x_tok.double().transpose(1, 2).reshape(B, C, side, side).requires_grad_(True)
    F.interpolate(a64, scale_factor=factor, mode="bilinear", align_corners=False).backward(dy.double().abs())
    terms = a64.grad.flatten(2).transpose(1, 2)                             # sum of w |dy| (the weights are >= 0)
    err = (grads[0].double() - want).abs()
    bound = U[dtype] * want.abs() + 2.0 ** -20 * terms + SUB[dtype]
    assert bool((err <= bound).all()), f"max err {err.max().item():.3e}, worst ratio {(err / bound).max().item():.3f}"


@pytest.mark.parametrize("dtype", DTYPES)
def test_clip_self_attention_backward_into_one_qkv_gradient(dtype):
    """4 images x 16 heads x hd 64 over T = 257 tokens, non-causal, q / k / v slices of the fused projection."""
    from mm_interleaved_b200 import autograd_ops, ops
    B, T, H, hd = 4, 257, 16, 64
    g = _gen(257)
    qkv = torch.randn(B, T, 3, H, hd, device=DEV, generator=g).to(dtype)
    d_out = torch.randn(B, T, H * hd, device=DEV, generator=g).to(dtype)
    x = qkv.clone().requires_grad_(True)
    out = autograd_ops.attention(x, causal=False)
    with torch.no_grad():
        assert torch.equal(out, ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], causal=False).reshape(B, T, H * hd))
    out.backward(d_out)
    assert x.grad.shape == qkv.shape and x.grad.is_contiguous()
    r = qkv.double().requires_grad_(True)
    q, k, v = r[:, :, 0], r[:, :, 1], r[:, :, 2]
    p = torch.softmax(torch.einsum("bqhd,bkhd->bhqk", q, k) * hd ** -0.5, -1)
    torch.einsum("bhqk,bkhd->bqhd", p, v).reshape(B, T, H * hd).backward(d_out.double())
    for i, name in enumerate(("dQ", "dK", "dV")):
        want = r.grad[:, :, i]
        err = (x.grad[:, :, i].double() - want).abs().max().item()
        assert err <= ATTN_TOL[dtype] * want.abs().max().item(), f"{name}: max err {err:.3e}"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("which", ["injector", "extractor"])
def test_msda_backward_at_the_adapter_shapes(which, dtype):
    from mm_interleaved_b200.functions import MSDeformAttnFunction
    shapes, Lq = ([(32, 32), (16, 16), (8, 8)], 256) if which == "injector" else ([(16, 16)], 1344)
    v, s, st, loc, a = make_msda_inputs(2, shapes, 16, 32, Lq, 4, seed=7, loc_mode="clustered", dtype=dtype)
    go = torch.randn((2, Lq, 16 * 32), generator=torch.Generator().manual_seed(3)).to(dtype)
    xs = [t.to(DEV, dtype).requires_grad_(True) for t in (v, loc, a)]
    MSDeformAttnFunction.apply(xs[0], s.to(DEV), st.to(DEV), xs[1], xs[2], 1).backward(go.to(DEV))
    rs = [t.double().requires_grad_(True) for t in (v, loc, a)]
    msda_core_pytorch(rs[0], s, rs[1], rs[2]).backward(go.double())
    # a point exactly at pixel coordinate -1 (16-bit locations reach it: loc = -1/(2 W)) is out of range for the
    # reference's CUDA op and this kernel (cuh:291, h_im > -1), so its location gradient is 0; the PyTorch core's
    # grid_sample takes the one-sided derivative into row / column 0 there.  Those points are compared as zeros.
    hw = torch.tensor(shapes, dtype=torch.float64)
    pix = loc.double() * torch.stack([hw[:, 1], hw[:, 0]], -1)[:, None, :] - 0.5
    edge = (pix == -1).any(-1, keepdim=True).expand_as(loc)
    assert bool((xs[1].grad.cpu()[edge] == 0).all())
    rs[1].grad[edge] = 0
    for x, r, name in zip(xs, rs, ("value", "loc", "attn")):
        err = (x.grad.double().cpu() - r.grad).abs().max()
        assert err <= 2e-2 * r.grad.abs().max() + 1e-7, (name, err.item(), r.grad.abs().max().item())


def _tokenizer(dtype, num_queries=None):
    """The fixture's tokenizer with its seeded weights; ``num_queries`` overrides the Q-Former's 8 queries (then the
    weights are seeded for that layout and not checked against the fixture)."""
    from mm_interleaved_b200 import visual_tokenizer as vt
    c = ADAPTER_GRAD_TINY
    pc = dict(c["perceiver"], **({} if num_queries is None else dict(num_queries=num_queries)))
    tok = vt.VisualTokenizer(clip_config=vt.CLIPVisionConfigLite(**c["clip"]), perceiver_config=pc,
                             llm_hidden_size=c["llm_hidden_size"], grid_size=c["grid_size"])
    sd = tokenizer_state_dict(tok.state_dict(), seed=WEIGHT_SEED)
    z = np.load(os.path.join(GOLDEN, "adapter_grad_tiny.npz"))
    if num_queries is None:
        assert sorted(sd.keys()) == [str(k) for k in z["keys"]]
        chk = float(sum(v.double().sum() for v in sd.values()))
        assert abs(chk - float(z["checksum"])) <= 1e-6 * max(1.0, abs(chk))
    tok.load_state_dict(sd, strict=True)
    return tok.freeze_like_reference().to(DEV, dtype).eval(), z


def _tokenizer_grads(tok, dtype, proj=None):
    images, golden_proj = adapter_grad_inputs()
    proj = golden_proj if proj is None else proj
    tok.zero_grad(set_to_none=True)
    outs = flat_outputs(tok(images.to(DEV, dtype)))
    sum((outs[k].double() * proj[k].to(DEV)).sum() for k in OUTPUTS).backward()
    return {k: o.detach() for k, o in outs.items()}, {n: p.grad.clone() for n, p in tok.named_parameters() if p.requires_grad}


def _grad_class(name):
    """The bound class of a trainable tensor (ADAPTER_TOL)."""
    if "sampling_offsets" in name or "query_norm" in name:
        return "location"
    if ".adapter_spm.stem." in name:
        return "pool"
    return "rest"


@pytest.mark.parametrize("dtype", DTYPES)
def test_tokenizer_gradients_match_reference_golden(dtype, deterministic_cudnn, no_tf32):
    from tests.golden.make_adapter_grad import SPM_STAGES, retain_stage_grads
    tok, z = _tokenizer(dtype)
    stages = retain_stage_grads(tok.encoder.vision_model.adapter_spm)
    outs, grads = _tokenizer_grads(tok, dtype)
    assert sorted(grads) == [str(n) for n in z["trainable"]]
    for k in OUTPUTS:
        want = torch.from_numpy(z[f"out/{k}"]).double()
        assert float((sample(outs[k].double().cpu()) - want).norm() / want.norm()) <= ADAPTER_TOL["rest"][dtype], k
    rel = {}
    for n, g in grads.items():
        assert bool(torch.isfinite(g).all()), n
        ref = torch.from_numpy(z[f"grad/{n}"]).double()
        # the k_norm bias shifts every score of a query by one constant, which the softmax removes: its exact gradient is
        # 0, so the error is measured against the scale of the sibling k_norm.weight gradient (as in the Q-Former test).
        # The key bias before k_norm cancels the same way except through k_norm's per-token Jacobian (the softmax makes
        # the keys' gradients sum to zero), so it is measured against the key weight's gradient likewise.
        sibling = n.endswith("k_norm.bias") or n.endswith("attention.key.bias")
        scale = torch.from_numpy(z[f"grad/{n[:-4]}weight"]).norm() if sibling else ref.norm()
        rel[n] = float((sample(g.double().cpu()) - ref).norm()) / max(float(scale), 1e-30)
    # per stage: the gradient arriving at the spatial prior module's outputs, against the reference's
    for k in SPM_STAGES:
        ref = torch.from_numpy(z[f"stage/{k}"]).double()
        rel[f"stage/{k}"] = float((sample(stages[k].grad.double().cpu()) - ref).norm() / ref.norm())
    for cls in ("location", "pool", "rest"):
        errs = sorted(((e, n) for n, e in rel.items() if _grad_class(n) == cls), reverse=True)
        print(f"adapter grads {dtype} {cls}: {len(errs)} tensors, median {np.median([e for e, _ in errs]):.1e}, largest "
              + ", ".join(f"{n} {e:.1e}" for e, n in errs[:10]))
    print(f"adapter grads {dtype} stages: " + ", ".join(f"{k} {rel['stage/' + k]:.1e}" for k in SPM_STAGES))
    rest = [e for n, e in rel.items() if _grad_class(n) == "rest"]
    assert float(np.median(rest)) <= QFORMER_TOL[dtype], f"median {np.median(rest):.2e}"
    bad = {n: f"{e:.2e}" for n, e in rel.items() if e > ADAPTER_TOL[_grad_class(n)][dtype]}
    assert not bad, f"relative errors above their class bound: {bad}"


def _spm64(spm, x, routing):
    """The spatial prior module in float64 (torch ops; the LayerNorm is over the channel dim), on float64 copies of its
    parameters.  Returns (outputs, {name: float64 parameter}); appends to ``routing`` the ReLU masks and the max-pool
    indices, in order."""
    params = {n: p.detach().double().requires_grad_(True) for n, p in spm.named_parameters()}

    def run(prefix, seq, x):
        for i, m in enumerate(seq):
            n = f"{prefix}.{i}"
            if isinstance(m, torch.nn.Conv2d):
                x = F.conv2d(x, params[n + ".weight"], params.get(n + ".bias"), m.stride, m.padding)
            elif isinstance(m, torch.nn.ReLU):
                routing.append(x > 0)
                x = F.relu(x)
            elif isinstance(m, torch.nn.MaxPool2d):
                x, idx = F.max_pool2d(x, 3, 2, 1, return_indices=True)
                routing.append(idx)
            else:
                x = F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), params[n + ".weight"], params[n + ".bias"],
                                 m.eps).permute(0, 3, 1, 2)
        return x

    c1 = run("stem", spm.stem, x)
    c2 = run("conv2", spm.conv2, c1)
    c3 = run("conv3", spm.conv3, c2)
    c4 = run("conv4", spm.conv4, c3)
    outs = [F.conv2d(c, params[f"fc{i}.weight"], params[f"fc{i}.bias"]) for i, c in enumerate((c1, c2, c3, c4), 1)]
    return outs, params


@pytest.mark.parametrize("dtype", DTYPES)
def test_spm_backward_per_stage(dtype, deterministic_cudnn, no_tf32):
    """The spatial prior module alone, the fixture's weights and images, seeded output gradients, against float64.  With
    its ReLU gates and max-pool choices taken from the float64 forward, every gradient is within the Q-Former's bound:
    the module's backward is right.  With its own 16-bit forward, values within rounding of zero switch their ReLU gate
    and windows whose two largest values are within rounding of each other send their gradient to another pixel; that is
    where the stem's error in the golden comparison enters."""
    tok, _ = _tokenizer(dtype)
    vm = tok.encoder.vision_model
    spm = vm.adapter_spm
    images, _ = adapter_grad_inputs()
    with torch.no_grad():
        x = (images.to(DEV, dtype) - tok.clip_mean.to(dtype)) / tok.clip_std.to(dtype)
        n = vm.config.image_size // vm.config.patch_size * 16
        x = F.interpolate(x, size=(n, n), mode="bilinear", align_corners=False)
    routing = []
    outs64, p64 = _spm64(spm, x.double(), routing)
    g = torch.Generator(device=DEV).manual_seed(11)
    dys = [torch.randn(o.shape, device=DEV, generator=g, dtype=torch.float64) for o in outs64]
    sum((o * d).sum() for o, d in zip(outs64, dys)).backward()

    def grads16(forced):
        spm.zero_grad(set_to_none=True)
        route = iter(routing)

        def run(seq, h):
            for m in seq:
                if isinstance(m, torch.nn.MaxPool2d):
                    idx = next(route)
                    h = h.flatten(2).gather(2, idx.flatten(2)).view(idx.shape) if forced else m(h)
                elif isinstance(m, torch.nn.ReLU):
                    gate = next(route)
                    h = h * gate.to(h.dtype) if forced else m(h)
                else:
                    h = m(h)
            return h
        c1 = run(spm.stem, x)
        c2 = run(spm.conv2, c1)
        c3 = run(spm.conv3, c2)
        c4 = run(spm.conv4, c3)
        outs = [spm.fc1(c1), spm.fc2(c2), spm.fc3(c3), spm.fc4(c4)]
        sum((o.double() * d).sum() for o, d in zip(outs, dys)).backward()
        return {n: float((p.grad.double() - p64[n].grad).norm() / p64[n].grad.norm()) for n, p in spm.named_parameters()}

    with torch.no_grad():
        pooled = spm.stem[:-1](x)
        _, idx16 = F.max_pool2d(pooled, 3, 2, 1, return_indices=True)
    moved = float((idx16 != routing[3]).double().mean())
    natural, forced = grads16(False), grads16(True)
    print(f"spm {dtype}: max-pool windows routed differently from float64: {moved:.2%}; largest error with its own "
          f"routing {max(natural.values()):.1e} ({max(natural, key=natural.get)}), with the float64 gates and routing "
          f"{max(forced.values()):.1e} ({max(forced, key=forced.get)}); "
          + ", ".join(f"{n} {natural[n]:.1e}/{forced[n]:.1e}" for n in natural))
    assert moved > 0
    bad = {n: f"{e:.2e}" for n, e in forced.items() if e > QFORMER_TOL[dtype]}
    assert not bad, f"SPM gradients with the float64 gates and routing above {QFORMER_TOL[dtype]}: {bad}"
    assert max(v for n, v in natural.items() if n.startswith("stem.")) <= ADAPTER_TOL["pool"][dtype]
    assert max(v for n, v in natural.items() if not n.startswith("stem.")) <= ADAPTER_TOL["rest"][dtype]


def test_tokenizer_outputs_are_bit_identical_under_autograd(deterministic_cudnn):
    """Adapter and head trainable: the forward under autograd returns the no_grad outputs bit for bit, and the no_grad
    path equals a fully frozen tokenizer's; two forward + backward passes give bit-identical gradients.  32 queries: the
    Q-Former head's inference attention takes another kernel below 16 query rows, so its training forward matches it
    bit for bit only from 16 rows on (tests/test_qformer_bwd_gpu.py)."""
    tok, _ = _tokenizer(torch.bfloat16, num_queries=32)
    images, _ = adapter_grad_inputs()
    images = images.to(DEV, torch.bfloat16)
    with torch.no_grad():
        ref = flat_outputs(tok(images))
    got = flat_outputs(tok(images))
    assert got["ms0"].requires_grad and got["vis_embed"].requires_grad
    for k in OUTPUTS:
        assert torch.equal(got[k].detach(), ref[k]), k
    trainable = {n for n, p in tok.named_parameters() if p.requires_grad}
    tok.requires_grad_(False)
    with torch.no_grad():
        frozen = flat_outputs(tok(images))
    for k in OUTPUTS:
        assert torch.equal(frozen[k], ref[k]), k
    for n, p in tok.named_parameters():
        p.requires_grad_(n in trainable)
    g = torch.Generator().manual_seed(8)
    proj = {k: torch.randn(ref[k].shape, generator=g, dtype=torch.float64) for k in OUTPUTS}
    _, a = _tokenizer_grads(tok, torch.bfloat16, proj)
    _, b = _tokenizer_grads(tok, torch.bfloat16, proj)
    for n in a:
        assert torch.equal(a[n], b[n]), n


def test_trainable_clip_attention_weight_raises():
    tok, _ = _tokenizer(torch.bfloat16)
    tok.encoder.vision_model.encoder.layers[3].self_attn.k_proj.weight.requires_grad_(True)
    images, _ = adapter_grad_inputs()
    with pytest.raises(RuntimeError, match="CLIPAttention: the CLIP q / k / v projections have no weight gradient"):
        tok(images.to(DEV, torch.bfloat16))


def test_mm_interleaved_loss_backward_trains_the_adapter(deterministic_cudnn):
    """Reference freezing (adapter + head trainable, CLIP frozen): ``forward(...)["loss"].backward()`` equals the same
    loss spelled out at module level, gradient for gradient; a fully trainable encoder still raises."""
    from tests.test_mm_interleaved_gpu import _batch, _build
    model, _ = _build()
    model = model.to(torch.bfloat16).freeze_like_reference()
    ids, images, nimg, mask = _batch()
    batch = dict(text_ids=ids.to(DEV), image_tensors=images.to(DEV), num_image_per_seq=nimg.to(DEV),
                 attention_mask=mask.to(DEV), meta={"dataset_name": "synthetic"})
    with pytest.raises(RuntimeError, match="the visual tokenizer has no backward"):
        model(**batch)
    model.visual_tokenizer.freeze_like_reference()
    # at the reference's initialisation injector gamma and the MSDA offset / weight projections are zero, which leaves the
    # injectors and the query norms without gradient: make them non-zero
    from mm_interleaved_b200.visual_tokenizer import MSDeformAttn
    g = torch.Generator(device=DEV).manual_seed(5)
    with torch.no_grad():
        for blk in model.visual_tokenizer.encoder.vision_model.adapter_interactions:
            blk.injector.gamma.fill_(0.5)
        for mod in model.visual_tokenizer.encoder.modules():
            if isinstance(mod, MSDeformAttn):
                for w in (mod.sampling_offsets.weight, mod.attention_weights.weight):
                    w.copy_(0.02 * torch.randn(w.shape, device=DEV, generator=g))

    model(**batch)["loss"].backward()
    trainable = [(n, p) for n, p in model.named_parameters()
                 if p.requires_grad and n.split(".")[0] in ("mm_decoder", "text_decoder", "soi_token", "visual_tokenizer")]
    names = {n for n, _ in trainable}
    adapter = {n for n in names if n.startswith("visual_tokenizer.encoder.")}
    assert adapter and all(".vision_model.adapter" in n for n in adapter)
    for part in ("adapter_spm.stem.0.weight", "injector.gamma", "extractor.ffn.dwconv.dwconv.weight", "adapter_level_embed", "extra_extractors.1.attn.value_proj.weight", "perceiver_resampler.queries"):
        assert any(n.endswith(part) for n in names), part
    # the largest multi-scale map (16^2 here) is read only through c1 = adapter_up(c2) + spm.fc1(stem); this model's
    # decoder reads the 8^2, 4^2 and 2^2 maps (spatial_shapes [8, 4, 2]), so those two layers get no gradient, as in the
    # reference (the golden test covers them)
    unread = {n for n in adapter if ".adapter_up." in n or ".adapter_spm.fc1." in n}
    assert unread and all(p.grad is None for n, p in trainable if n in unread)
    got = {n: p.grad.clone() for n, p in trainable if n not in unread}
    assert all(g is not None and bool(torch.isfinite(g).all()) for g in got.values())
    zero = [n for n in adapter - unread if not float(got[n].abs().max()) > 0]
    assert not zero, f"adapter tensors without gradient: {zero}"
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
        assert (p.grad is None) if n in unread else torch.equal(p.grad, got[n]), n
