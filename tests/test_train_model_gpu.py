"""GPU tests of the text-loss training path through the Llama-MMFS decoder (the reference's freezing: only the
``llama_cross_attn`` blocks trainable).

The tiny decoder is LLAMA_TC-shaped (hidden 256 in two heads of 128, 3 layers with cross-attention in layers 0 and 2,
T = 200, 3 images, batch entry 1 left-padded by 5).  Its loss is the cross-entropy of a fixed random head at the
non-pad positions only, so the oracle's rule for fully masked rows (a uniform softmax, where the kernel returns 0)
cannot reach it.  The gradients of every trainable parameter, of ``inputs_embeds`` and of ``vision_hidden_states`` are
compared with fp32 autograd through the CPU oracle (oracle/llama.py + oracle/mmfs.py) on the same 16-bit weights and
inputs, as relative Frobenius-norm errors per tensor.  (fp32, not float64: in float64 the oracle's additive mask
finfo.min + finfo.min overflows to -inf on the fully masked rows, which turns them into NaN, and masked keys then carry
0 * NaN into valid rows; fp32 rounding is far below the 16-bit bounds.)  The bounds, 6e-2 (bf16) / 1e-2 (fp16), are those of the
decoder's forward in tests/test_llama_gpu.py (4e-2 of max |ref| in bf16) plus the backward's own 16-bit roundings of the
same size: every activation and gradient between layers is stored in the element type.  The oracle samples the
MMFS features at sampling locations rounded to the element type, as the reference's 16-bit model does.
``sampling_offsets`` alone has a looser bound, stated where it is checked."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"

from tests.golden.make_golden import LLAMA_TC, LLAMA_TINY, llama_inputs, seeded_state_dict  # noqa: E402

GRAD_TOL = {torch.bfloat16: 6e-2, torch.float16: 1e-2}
CFG = {**LLAMA_TINY, "max_position_embeddings": 256}


def _model(dtype, checkpointing=False):
    from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, LlamaModel
    model = LlamaModel(LlamaMMFSConfig(**CFG))
    sd = seeded_state_dict(model.state_dict(), seed=4242)
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV, dtype).train()
    for name, p in model.named_parameters():              # mm_interleaved.py:74-78
        p.requires_grad_("llama_cross_attn" in name)
    model.gradient_checkpointing = checkpointing
    return model


def _inputs(dtype):
    c = LLAMA_TC
    embeds, vision, mask, pos, cross = llama_inputs(LLAMA_TINY, c["B"], c["T"], c["n_img"], seed=c["seed"], left_pad=c["left_pad"])
    g = torch.Generator().manual_seed(5)
    head = torch.randn(LLAMA_TINY["hidden_size"], 64, generator=g) * 0.1
    target = torch.randint(0, 64, (c["B"], c["T"]), generator=g).masked_fill(mask == 0, -100)
    return embeds.to(dtype), vision.to(dtype), mask, pos, cross, head, target


def _run(model, dtype):
    embeds, vision, mask, pos, cross, head, target = _inputs(dtype)
    e = embeds.to(DEV).requires_grad_(True)
    v = vision.to(DEV).requires_grad_(True)
    out = model(inputs_embeds=e, attention_mask=mask.to(DEV), position_ids=pos.to(DEV), vision_hidden_states=v,
                cross_attention_mask=cross.to(DEV), use_cache=False).last_hidden_state
    loss = F.cross_entropy((out.float() @ head.to(DEV)).transpose(1, 2), target.to(DEV))
    loss.backward()
    grads = {n: p.grad for n, p in model.named_parameters() if p.requires_grad}
    grads["inputs_embeds"], grads["vision_hidden_states"] = e.grad, v.grad
    return loss.detach(), grads


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_decoder_gradients_match_fp32_oracle(dtype):
    from oracle.llama import llama_model_ref
    model = _model(dtype)
    loss, grads = _run(model, dtype)
    assert len(grads) == 2 + sum(1 for n, _ in model.named_parameters() if "llama_cross_attn" in n)

    embeds, vision, mask, pos, cross, head, target = _inputs(dtype)
    sd = {n: p.detach().float().cpu().requires_grad_("llama_cross_attn" in n) for n, p in model.named_parameters()}
    e, v = embeds.float().requires_grad_(True), vision.float().requires_grad_(True)
    ocfg = dict(eps=CFG["rms_norm_eps"], n_heads=CFG["num_attention_heads"], n_layers=CFG["num_hidden_layers"],
                spatial_shapes=[(s, s) for s in CFG["spatial_shapes"]])
    # the reference's bf16 / fp16 model rounds the sampling locations to the element type (loc.to(value.dtype),
    # mmfs.py:250) and autograd passes the cast through; the fp32 oracle would keep them in fp32, and bilinear
    # sampling's location gradient jumps where a point crosses a pixel boundary
    import oracle.mmfs as omm
    core = omm.msda_core_pytorch

    def core_16bit_locations(value, shapes, loc, attn):
        return core(value, shapes, loc + (loc.to(dtype).to(loc.dtype) - loc).detach(), attn)
    omm.msda_core_pytorch = core_16bit_locations
    try:
        ref_out, _ = llama_model_ref(sd, e, mask, pos, v, cross, ocfg)
    finally:
        omm.msda_core_pytorch = core
    ref_loss = F.cross_entropy((ref_out @ head).transpose(1, 2), target)
    ref_loss.backward()
    ref = {n: t.grad for n, t in sd.items() if t.requires_grad}
    ref["inputs_embeds"], ref["vision_hidden_states"] = e.grad, v.grad

    assert abs(float(loss) - float(ref_loss.detach())) <= GRAD_TOL[dtype] * abs(float(ref_loss.detach()))
    assert set(grads) == set(ref)
    rel = {n: float((grads[n].double().cpu() - r).norm()) / max(float(r.norm()), 1e-30) for n, r in ref.items()}
    # sampling_offsets: its gradient is the location gradient of bilinear sampling, which jumps where a point crosses a
    # pixel boundary.  The oracle samples at the same 16-bit-rounded locations (above), but the offsets feeding them are
    # computed in 16 bits here and in fp32 there, so a few rounded locations still differ by one step: measured 9.3e-2
    # (bf16) / 2.0e-2 (fp16) on this case, where every other tensor is within GRAD_TOL; bound 3 x GRAD_TOL.
    tol = {n: GRAD_TOL[dtype] * (3 if ".sampling_offsets." in n else 1) for n in rel}
    bad = {n: f"{e:.2e}" for n, e in rel.items() if e > tol[n]}
    assert not bad, f"relative errors above the bound: {bad}; all: { {n: f'{e:.1e}' for n, e in rel.items()} }"
    assert float(ref["inputs_embeds"][1, :LLAMA_TC["left_pad"]].abs().max()) == 0.0
    assert float(grads["inputs_embeds"][1, :LLAMA_TC["left_pad"]].abs().max()) == 0.0


def test_gradient_checkpointing_gives_identical_gradients():
    """Same deterministic kernels on the same inputs in the recomputation: bit-identical gradients."""
    loss_a, a = _run(_model(torch.bfloat16), torch.bfloat16)
    loss_b, b = _run(_model(torch.bfloat16, checkpointing=True), torch.bfloat16)
    assert torch.equal(loss_a, loss_b)
    for n in a:
        assert torch.equal(a[n], b[n]), n


def test_documented_errors_under_autograd():
    from mm_interleaved_b200.llama_mmfs import LlamaMMFSConfig, LlamaModel
    embeds, vision, mask, pos, cross, _, _ = _inputs(torch.bfloat16)
    kw = dict(attention_mask=mask.to(DEV), position_ids=pos.to(DEV), cross_attention_mask=cross.to(DEV))
    model = _model(torch.bfloat16)
    with pytest.raises(RuntimeError, match="without a KV cache"):
        model(inputs_embeds=embeds.to(DEV), vision_hidden_states=vision.to(DEV), use_cache=True, **kw)
    m32 = _model(torch.float32)
    with pytest.raises(RuntimeError, match="bf16 / fp16 only"):
        m32(inputs_embeds=embeds.float().to(DEV), vision_hidden_states=vision.float().to(DEV), use_cache=False, **kw)
    m64 = LlamaModel(LlamaMMFSConfig(**{**CFG, "num_attention_heads": 4})).to(DEV, torch.bfloat16)
    with pytest.raises(RuntimeError, match="head dim 128"):
        m64(inputs_embeds=embeds.to(DEV), vision_hidden_states=vision.to(DEV), use_cache=False, **kw)
    with torch.no_grad():      # the inference path is untouched by the trainable flags
        model(inputs_embeds=embeds.to(DEV), vision_hidden_states=vision.to(DEV), use_cache=False, **kw)


def _mm_batch(model):
    from tests.test_mm_interleaved_gpu import _batch
    ids, images, nimg, mask = _batch()
    return dict(text_ids=ids.to(DEV), image_tensors=images.to(DEV), num_image_per_seq=nimg.to(DEV),
                attention_mask=mask.to(DEV), meta={"dataset_name": "synthetic"})


def test_mm_interleaved_loss_backward_matches_the_decoder_level_computation():
    from tests.test_mm_interleaved_gpu import _build
    model, _ = _build()
    model = model.to(torch.bfloat16).freeze_like_reference()
    batch = _mm_batch(model)
    with pytest.raises(RuntimeError, match="visual tokenizer has no backward"):
        model(**batch)
    model.visual_tokenizer.requires_grad_(False)
    model._has_image_loss = lambda: True
    with pytest.raises(RuntimeError, match="image-decoder loss has no backward"):
        model(**batch)
    del model._has_image_loss

    model(**batch)["loss"].backward()
    trainable = [(n, p) for n, p in model.named_parameters()          # context_feat_proj: the image loss's only
                 if p.requires_grad and n.split(".")[0] in ("mm_decoder", "text_decoder", "soi_token")]
    names = {n for n, _ in trainable}
    assert "soi_token" in names and "text_decoder.head_new.weight" in names
    assert all("llama_cross_attn" in n for n in names if n.startswith("mm_decoder."))
    got = {n: p.grad.clone() for n, p in trainable}
    assert all(g is not None and bool(torch.isfinite(g).all()) for g in got.values())
    assert float(got["soi_token"].abs().max()) > 0 and float(got["mm_decoder.layers.0.llama_cross_attn.gate"].abs().max()) > 0
    model.zero_grad(set_to_none=True)

    # the same loss spelled out at the decoder level
    nimg = batch["num_image_per_seq"].reshape(-1)
    vis = model.visual_tokenizer(batch["image_tensors"].to(torch.bfloat16))
    mm_embeds, cross, feats = model.prepare(batch["text_ids"], vis, nimg, int(nimg.max()))
    hidden = model.mm_decoder(inputs_embeds=mm_embeds, attention_mask=batch["attention_mask"], vision_hidden_states=feats,
                              cross_attention_mask=cross, use_cache=False).last_hidden_state
    logits = model.text_decoder.logits(hidden)
    gt = model._prepare_gt_text_ids(batch["text_ids"], batch["attention_mask"], 0, None, batch["meta"])
    F.cross_entropy(logits[:, :-1].float().transpose(1, 2), gt.contiguous()).backward()
    for n, p in trainable:
        assert torch.equal(p.grad, got[n]), n
