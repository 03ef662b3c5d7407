"""GPU tests of ``MMInterleaved.generate_interleaved`` (interleaved.py) on a tiny fp32 model with a tiny VAE decoder,
against a test-side restatement of the reference's ``inference.py::inference_all`` loop: ``model.generate(mode=...)``
per turn over the whole context, ``update_texts`` on tensors and ``update_image`` through PIL on the host.

Every text turn's ids equal the loop's; every image is within the tolerance the generate-images test uses against a
recomputation; the final text ids, attention mask and image count are equal.  The final image tensor holds exactly the
PIL re-entry of the session's own images, and equals the loop's up to one quantisation step where the two runs'
images straddle a rounding boundary (their fp32 values differ in the last bits: the session prefills in chunks over a
cache, the loop from scratch)."""
import numpy as np
import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_TOK, R, SIZE = 4, 48, 128          # <image> ids per image, tokenizer input size, generated image size (128 -> 64 -> 48)
ST = dict(bos_token_id=1, eos_token_id=2, pad_token_id=0, soi_token_id=63, image_token_id=62)
IMG_TOL = dict(rtol=1e-3, atol=1e-4)


class TinyTokenizer(nn.Module):
    """Stands in for the visual tokenizer: ``N_TOK`` embeddings and four feature maps (16, 8, 4, 2) per image, each a
    smooth function of the image, so a re-entered image changes what the decoder sees."""

    def __init__(self, hidden, channels):
        super().__init__()
        self.proj = nn.Linear(3, hidden)
        self.maps = nn.Linear(3, channels)
        self.calls, self.images = 0, 0

    def forward(self, image):
        self.calls += 1
        self.images += image.shape[0]
        tok = nn.functional.adaptive_avg_pool2d(image, (2, 2)).flatten(2).transpose(1, 2)        # (n, 4, 3)
        feats = [torch.tanh(self.maps(nn.functional.adaptive_avg_pool2d(image, s).permute(0, 2, 3, 1)) * 3)
                 .permute(0, 3, 1, 2).contiguous() for s in (16, 8, 4, 2)]
        return {"vis_embed": torch.tanh(self.proj(tok * 4 - 2)), "multiscale_features": feats}


def build(seed=77):
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    from mm_interleaved_b200.mm_interleaved import ImageDecoder, MMInterleaved
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    from tests.golden.make_golden import LLAMA_TINY, seeded_state_dict
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)
    cfg = m.LlamaMMFSConfig(**LLAMA_TINY)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(64, 128), layers_per_block=1, attention_head_dim=(2, 4),
                                        cross_attention_dim=96)
    net = m.MMFSNet(cfg.image_embed_dim, (64, 128), 1, downsample_factor=2, spatial_shapes=[16, 8, 4, 2])
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.2)
    vae = AutoencoderKL(block_out_channels=(32, 32, 64, 64), layers_per_block=1)
    dec = ImageDecoder(perceiver_config=dict(num_queries=7, hidden_size=96, encoder_hidden_size=cfg.hidden_size,
                                             num_hidden_layers=2, num_attention_heads=4, intermediate_size=192,
                                             cross_attention_frequency=1, qk_normalization=True),
                       seq_len=7, embed_dim=96, unet=unet, mmfs_module=net, image_size=SIZE, vae=vae)
    model = MMInterleaved(llm_config=cfg, txt_vocab_size=cfg.vocab_size, seq_len=128, special_token_dict=ST,
                          num_img_token=N_TOK, image_embed_dim=cfg.image_embed_dim,
                          cross_attention_frequency=cfg.cross_attention_frequency, spatial_shapes=cfg.spatial_shapes,
                          visual_tokenizer=TinyTokenizer(cfg.hidden_size, cfg.image_embed_dim), image_decoder=dec)
    sd = model.state_dict()
    keys = {k: v for k, v in sd.items() if k.startswith(("mm_decoder.", "text_decoder.", "soi_token", "context_feat"))}
    sd.update(seeded_state_dict(keys, seed=seed))
    model.load_state_dict(sd)
    return model.to(DEV).eval()


def sample(n_img=2, image_last=False, seed=3):
    """A load_annt_data-like sample: <bos>, text, and n_img images as <soi> + N_TOK <image>; with ``image_last`` the
    text ends with an image subsequence (a first image turn generates it)."""
    g = torch.Generator().manual_seed(seed)
    ids = [1]
    for _ in range(n_img):
        ids += torch.randint(3, 60, (5,), generator=g).tolist() + [63] + [62] * N_TOK
    if not image_last:
        ids += torch.randint(3, 60, (4,), generator=g).tolist()
    images = torch.rand((n_img, 3, R, R), generator=g)
    if image_last:
        images[-1] = 0.5
    ids = torch.tensor([ids])
    return dict(text_ids=ids.to(DEV), attention_mask=torch.ones_like(ids).to(DEV), image_tensors=images.to(DEV),
                num_image_per_seq=torch.tensor([n_img], device=DEV), target_image_idxs=torch.tensor([n_img - 1], device=DEV))


# ---- the reference loop, restated ------------------------------------------------------------------------------------
def pil_reentry(image):
    """update_image: tensor_to_pil, center_crop_arr(R) with PIL, float32 / 255 (utils/clip_sim_score.py,
    custom_datasets/utils.py)."""
    from PIL import Image
    arr = image.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8).numpy()
    pil = Image.fromarray(arr).convert("RGB")
    while min(*pil.size) >= 2 * R:
        pil = pil.resize(tuple(x // 2 for x in pil.size), resample=Image.BOX)
    scale = R / min(*pil.size)
    pil = pil.resize(tuple(round(x * scale) for x in pil.size), resample=Image.BICUBIC)
    arr = np.array(pil)
    cy, cx = (arr.shape[0] - R) // 2, (arr.shape[1] - R) // 2
    arr = arr[cy:cy + R, cx:cx + R].astype(np.float32).transpose([2, 0, 1]) / 255.0
    return torch.from_numpy(arr)


def reference_loop(model, inputs, generate_mode, num_iter, auto_end, force_gen_image_next, generator=None, **gen):
    inputs = {k: v.clone() for k, v in inputs.items()}
    turns, mode, stopped = [], generate_mode, False
    for _ in range(num_iter):
        out = model.generate(mode=mode, **inputs, generator=generator, **gen)
        if mode == "generate_texts":
            turns.append(("t", out["text_ids"]))
            t = out["text_ids"][0][1:]                                           # update_texts
            gen_image_next = False
            if t[-1] == ST["eos_token_id"]:
                t, stopped = t[:-1], True
            if force_gen_image_next and t[-1] != ST["soi_token_id"]:
                t = torch.cat((t, torch.tensor([ST["soi_token_id"]]).type_as(t)))
            if t[-1] == ST["soi_token_id"]:
                t = torch.cat((t, torch.tensor([ST["image_token_id"]] * N_TOK).type_as(t)))
                inputs["image_tensors"] = torch.cat([inputs["image_tensors"], torch.full((1, 3, R, R), 0.5, device=DEV)])
                inputs["target_image_idxs"] = inputs["target_image_idxs"] + 1
                inputs["num_image_per_seq"] = inputs["num_image_per_seq"] + 1
                gen_image_next = True
            inputs["text_ids"] = torch.cat((inputs["text_ids"], t[None].to(DEV)), dim=-1)
            inputs["attention_mask"] = torch.cat((inputs["attention_mask"], torch.ones_like(t[None]).to(DEV)), dim=-1)
            if gen_image_next:
                mode = "generate_images"
        else:
            turns.append(("i", out["image"]))
            inputs["image_tensors"][-1, ...] = pil_reentry(out["image"][0]).to(DEV)   # update_image
            mode = "generate_texts"
        if auto_end and stopped:
            break
    return turns, inputs


def compare(out, turns, inputs):
    assert len(out["turns"]) == len(turns)
    for got, (kind, want) in zip(out["turns"], turns):
        if kind == "t":
            assert got["mode"] == "generate_texts"
            assert torch.equal(got["text_ids"].cpu(), want.cpu()), (got["text_ids"], want)
        else:
            assert got["mode"] == "generate_images"
            torch.testing.assert_close(got["image"], want, **IMG_TOL)
    assert torch.equal(out["text_ids"].cpu(), inputs["text_ids"].cpu())
    assert torch.equal(out["attention_mask"].cpu(), inputs["attention_mask"].cpu())
    assert torch.equal(out["num_image_per_seq"].cpu(), inputs["num_image_per_seq"].reshape(-1).cpu())
    imgs = out["image_tensors"].cpu()
    assert imgs.shape == inputs["image_tensors"].shape
    diff = (imgs - inputs["image_tensors"].cpu()).abs()
    assert float(diff.max()) <= 1.0001 / 255 and float((diff > 0).float().mean()) < 1e-3, float(diff.max())


GEN = dict(max_length=6, min_length=2, num_inference_steps=3, guidance_scale=3.0, num_validation_images=1)


def test_greedy_text_image_text_image_matches_the_reference_loop():
    model = build()
    inputs = sample()
    gen = dict(GEN, num_beams=1)
    tok = model.visual_tokenizer
    tok.calls = tok.images = 0
    from mm_interleaved_b200 import generation
    spans, orig = [], generation._prefill

    def spy(m, p, past, vision):
        spans.append((p.prefix, p.mm_embeds.shape[1]))
        return orig(m, p, past, vision)

    generation._prefill = spy
    try:
        out = model.generate_interleaved(**{k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors",
                                                                   "num_image_per_seq")},
                                         num_iter=4, force_gen_image_next=True, return_session=True, **gen)
    finally:
        generation._prefill = orig
    assert [t["mode"] for t in out["turns"]] == ["generate_texts", "generate_images"] * 2
    # one tokenizer pass per image: the two inputs at once, then each generated image alone
    assert tok.images == int(out["num_image_per_seq"]) == 4 and tok.calls == 3
    # each position prefilled once: the chunks tile [0, cached)
    session = out.pop("session")
    assert spans[0][0] == 0 and all(a[1] == b[0] for a, b in zip(spans, spans[1:])) and spans[-1][1] == session.cached
    assert session.cached <= session.capacity
    turns, ref_inputs = reference_loop(model, inputs, "generate_texts", 4, False, True, **gen)
    compare(out, turns, ref_inputs)
    # the final slot holds exactly the PIL re-entry of the session's last image
    assert torch.equal(out["image_tensors"][-1].cpu(), pil_reentry(out["turns"][-1]["image"][0].clone()))

    # the cached hidden states equal a from-scratch prefill of the same context
    L = session.cached
    ids = torch.tensor([session.ids[:L]], device=DEV)
    n = int(out["num_image_per_seq"])
    with torch.no_grad():
        vis = model._tokenize(out["image_tensors"])
        mm, cross, feats = model.prepare(ids, vis, torch.tensor([n], device=DEV), n)
        full = model.mm_decoder(inputs_embeds=mm, attention_mask=torch.ones_like(ids), vision_hidden_states=feats,
                                cross_attention_mask=cross, use_cache=False, return_dict=True).last_hidden_state
    torch.testing.assert_close(session.hidden[:, :L], full, rtol=1e-3, atol=1e-4)


def test_image_turn_context_and_mmfs_features_equal_generate_images():
    model = build()
    inputs = sample(n_img=2, image_last=True)
    seen = []
    dec = model.image_decoder
    orig = dec.generate_images

    def spy(**kw):
        seen.append(kw)
        return orig(**kw)

    dec.generate_images = spy
    try:
        out = model.generate_interleaved(**{k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors",
                                                                   "num_image_per_seq")},
                                         generate_mode="generate_images", num_iter=1, **GEN)
        ref = model.generate(mode="generate_images", **inputs, **GEN)
    finally:
        dec.generate_images = orig
    got, want = seen
    torch.testing.assert_close(got["context_features"], want["context_features"], rtol=1e-3, atol=1e-4)
    assert torch.equal(got["context_attention_mask"], want["context_attention_mask"])
    assert torch.equal(got["mmfs_mask"], want["mmfs_mask"]) and int(got["mmfs_mask"].sum()) == 1
    for a, b in zip(got["mmfs_features"], want["mmfs_features"]):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(out["turns"][0]["image"], ref["image"], **IMG_TOL)


@pytest.mark.parametrize("graphs", [False, True])
def test_beam_search_turns_match_the_reference_loop(graphs):
    model = build()
    if graphs:
        model.enable_decode_graphs()
    inputs = sample()
    gen = dict(GEN, num_beams=5, max_length=5)
    kw = {k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors", "num_image_per_seq")}
    out = model.generate_interleaved(**kw, num_iter=3, force_gen_image_next=True, **gen)
    turns, ref_inputs = reference_loop(model, inputs, "generate_texts", 3, False, True, **gen)
    compare(out, turns, ref_inputs)


@pytest.mark.parametrize("graphs", [False, True])
def test_seeded_sampling_session_reproduces_itself(graphs):
    model = build()
    if graphs:
        model.enable_decode_graphs(True, sampling=True)
        model.enable_cuda_graphs()
    inputs = sample()
    gen = dict(GEN, num_beams=1, use_nucleus_sampling=True, top_p=0.9, repetition_penalty=1.3)
    kw = {k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors", "num_image_per_seq")}
    runs = [model.generate_interleaved(**kw, num_iter=3, force_gen_image_next=True,
                                       generator=torch.Generator(device=DEV).manual_seed(11), **gen) for _ in range(2)]
    a, b = runs
    assert [t["mode"] for t in a["turns"]] == ["generate_texts", "generate_images", "generate_texts"]
    for x, y in zip(a["turns"], b["turns"]):
        key = "text_ids" if x["mode"] == "generate_texts" else "image"
        assert torch.equal(x[key], y[key])
    assert torch.equal(a["text_ids"], b["text_ids"]) and torch.equal(a["image_tensors"], b["image_tensors"])
    if not graphs:                    # eager sampling draws like the loop's generate_texts from the same generator
        turns, ref_inputs = reference_loop(model, inputs, "generate_texts", 3, False, True,
                                           generator=torch.Generator(device=DEV).manual_seed(11), **gen)
        compare(a, turns, ref_inputs)


def test_auto_end_stops_at_eos():
    model = build()
    with torch.no_grad():                                        # eos wins once min_length allows it: at the last step
        model.text_decoder.head.bias[ST["eos_token_id"]] += 100.0
    inputs = sample()
    gen = dict(GEN, num_beams=1, max_length=4, min_length=3)
    kw = {k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors", "num_image_per_seq")}
    out = model.generate_interleaved(**kw, num_iter=4, auto_end=True, **gen)
    assert len(out["turns"]) == 1 and int(out["turns"][0]["text_ids"][0, -1]) == ST["eos_token_id"]
    turns, ref_inputs = reference_loop(model, inputs, "generate_texts", 4, True, False, **gen)
    compare(out, turns, ref_inputs)


def test_text_turns_without_soi_stay_text():
    model = build()
    with torch.no_grad():                                        # never <soi>: the text continues with text
        model.text_decoder.head_new.bias[ST["soi_token_id"] - 62] -= 100.0
    inputs = sample()
    gen = dict(GEN, num_beams=1)
    kw = {k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors", "num_image_per_seq")}
    out = model.generate_interleaved(**kw, num_iter=3, force_gen_image_next=False, **gen)
    assert [t["mode"] for t in out["turns"]] == ["generate_texts"] * 3
    turns, ref_inputs = reference_loop(model, inputs, "generate_texts", 3, False, False, **gen)
    compare(out, turns, ref_inputs)


def test_first_turn_generates_an_image():
    model = build()
    inputs = sample(n_img=2, image_last=True)
    gen = dict(GEN, num_beams=1)
    kw = {k: inputs[k] for k in ("text_ids", "attention_mask", "image_tensors", "num_image_per_seq")}
    tok = model.visual_tokenizer
    tok.calls = tok.images = 0
    out = model.generate_interleaved(**kw, generate_mode="generate_images", num_iter=3, force_gen_image_next=True, **gen)
    assert [t["mode"] for t in out["turns"]] == ["generate_images", "generate_texts", "generate_images"]
    assert tok.images == int(out["num_image_per_seq"]) == 3
    turns, ref_inputs = reference_loop(model, inputs, "generate_images", 3, False, True, **gen)
    compare(out, turns, ref_inputs)
