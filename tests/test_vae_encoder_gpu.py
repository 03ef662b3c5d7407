"""GPU tests of the image-decoder loss path: the one-sided-pad downsample convolution (csrc/conv_igemm_sm100.cu through
``ops.conv2d_down2x``), the SD-2.1 VAE encoder (vae_sd.py), ``StableDiffusion.forward``, ``ImageDecoder.forward`` and
``MMInterleaved.forward``'s ``loss_img``.

Per-kernel bound, as in test_vae_gpu.py: max |err| <= 2e-2 * max|ref| and mean |err| <= 2e-3 * max|ref| against fp32
``F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2)`` on the same rounded operands (cuDNN with TF32 off).  Whole models in
bf16 against the fp32 restatements get the UNet's full-width bound: max <= 6e-2 of max|ref|, relative RMS <= 3e-2."""
import pytest
import torch
import torch.nn.functional as F

from tests.image_loss_oracle import add_noise_ref, vae_encode_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _check(out, ref):
    err = (out.float() - ref).abs()
    scale = ref.abs().max()
    assert err.max() <= 2e-2 * scale, (err.max().item(), scale.item())
    assert err.mean() <= 2e-3 * scale, (err.mean().item(), scale.item())


def _rel(got, ref):
    err = got.float().cpu() - ref.float().cpu()
    return (err.abs().max() / ref.abs().max()).item(), (err.pow(2).mean().sqrt() / ref.float().pow(2).mean().sqrt()).item()


DOWN_CASES = [(1, 128, 512), (1, 256, 256), (1, 512, 128), (2, 128, 16)]     # B, C, H = W; the encoder's three + 8x8 out


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", range(len(DOWN_CASES)))
def test_conv2d_down2x_matches_pad_then_strided_conv(case, dtype):
    from mm_interleaved_b200 import ops
    B, C, H = DOWN_CASES[case]
    g = torch.Generator(device=DEV).manual_seed(100 + case)
    x = torch.randn((B, C, H, H), generator=g, device=DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    w = (torch.randn((C, C, 3, 3), generator=g, device=DEV) / (C * 9) ** 0.5).to(dtype)
    bias = torch.randn(C, generator=g, device=DEV).to(dtype)
    assert ops.conv2d_down2x_supported(x, w)
    out = ops.conv2d_down2x(x, w.permute(0, 2, 3, 1).contiguous(), bias)
    ref = F.conv2d(F.pad(x.float(), (0, 1, 0, 1)), w.float(), bias.float(), stride=2)
    assert out.shape == ref.shape == (B, C, H // 2, H // 2) and out.is_contiguous(memory_format=torch.channels_last)
    _check(out, ref)
    # the last output row / column are where the one-sided pad enters: held to the same bound on their own
    _check(out[..., -1, :], ref[..., -1, :])
    _check(out[..., :, -1], ref[..., :, -1])


def _seeded_vae(**kw):
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    torch.manual_seed(0)
    m = AutoencoderKL(with_encoder=True, **kw).eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "norm" in name:                                    # make the GroupNorm affine terms count
                p.add_(0.2 * torch.randn(p.shape, generator=g))
    return m


def test_whole_encoder_sd21_widths_fp32_and_bf16_against_oracle(monkeypatch):
    from mm_interleaved_b200 import ops
    m = _seeded_vae().to(DEV)
    x = torch.rand((1, 3, 512, 512), generator=torch.Generator().manual_seed(2)) * 2 - 1
    mean, logvar = vae_encode_ref({k: v.to(DEV) for k, v in m.state_dict().items()}, x.to(DEV))     # fp32, TF32 off
    assert mean.shape == (1, 4, 64, 64)

    p32 = m.encode(x.to(DEV)).latent_dist
    for got, ref in ((p32.mean, mean), (p32.logvar, logvar)):
        assert (got - ref).abs().max() <= 1e-3 * ref.abs().max(), ((got - ref).abs().max() / ref.abs().max()).item()

    m16 = m.to(torch.bfloat16)
    calls = {"conv2d": 0, "conv2d_down2x": 0}
    for name in calls:
        def counted(*a, _f=getattr(ops, name), _n=name, **k):
            calls[_n] += 1
            return _f(*a, **k)
        monkeypatch.setattr(ops, name, counted)
    before = ops.launch_counter[0]
    a = m16.encode(x.to(DEV)).latent_dist
    launches = ops.launch_counter[0] - before
    # 10 resnets x 2 convs + 2 shortcuts on the wgmma kernel, 3 downsamplers on the down2x entry
    assert calls == {"conv2d": 22, "conv2d_down2x": 3}, calls
    assert launches >= 25
    b = m16.encode(x.to(DEV)).latent_dist
    assert a.mean.dtype == torch.bfloat16 and torch.equal(a.mean, b.mean) and torch.equal(a.logvar, b.logvar)
    for name, got, ref in (("mean", a.mean, mean), ("logvar", a.logvar, logvar)):
        rel_max, rel_rms = _rel(got, ref)
        print(f"whole encoder bf16 {name} vs fp32 oracle: max {rel_max:.3e} of max|ref|, relative RMS {rel_rms:.3e}")
        assert rel_max <= 6e-2 and rel_rms <= 3e-2


def _tiny_sd(dtype=torch.float32):
    """Tiny UNet + MMFSNet of test_unet_oracle.py with a 4-level VAE (128 x 128 images -> 16 x 16 latents)."""
    from mm_interleaved_b200.mm_interleaved import StableDiffusion
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    from tests.test_unet_oracle import _tiny
    unet, net, _, ctx, feats, mask = _tiny()
    torch.manual_seed(1)
    vae = AutoencoderKL(block_out_channels=(32, 32, 64, 64), layers_per_block=1, with_encoder=True).eval()
    sd = StableDiffusion(unet=unet, mmfs_module=net, image_size=128, vae=vae, vae_encode_mini_bs=1).to(DEV, dtype)
    image = torch.rand((2, 3, 128, 128), generator=torch.Generator().manual_seed(12))
    return sd, image, ctx, feats, mask


def _sd_forward_ref(sd, image, ctx, feats, mask, seed, dtype):
    """sd.py:240-316 restated: the oracle encode per chunk of one image, the draws replayed from an equally seeded
    generator in the model's order and dtypes, the float64 ``add_noise``, the oracle UNet with the MMFSNet oracle hook,
    and the MSE.  Weights (rounded to ``dtype``) in fp32 on the CPU."""
    from oracle.sd_mmfs import mmfsnet_ref
    from oracle.unet import unet_forward_ref
    f32 = lambda m: {k: v.detach().float().cpu() for k, v in m.state_dict().items()}
    vsd, usd, nsd = f32(sd.vae), f32(sd.unet), f32(sd.mmfs_module)
    g = torch.Generator(device=DEV).manual_seed(seed)
    parts = []
    for i in range(image.shape[0]):
        mean, logvar = vae_encode_ref(vsd, ((image[i:i + 1].float() - 0.5) / 0.5).to(dtype))
        eps = torch.randn(mean.shape, generator=g, device=DEV, dtype=dtype).float().cpu()
        parts.append(mean + torch.exp(0.5 * logvar) * eps)
    latents = torch.cat(parts) * 0.18215
    noise = torch.randn(latents.shape, generator=g, device=DEV, dtype=dtype).float().cpu()
    t = torch.randint(0, 1000, (latents.shape[0],), generator=g, device=DEV).cpu()
    acp = sd.noise_scheduler.alphas_cumprod.to(dtype)
    noisy = add_noise_ref(acp, latents, noise, t).float()
    hook = lambda s, res, f, mk: mmfsnet_ref(nsd, s, list(res), f, mk, downsample_factor=2, n_down=len(res))
    pred = unet_forward_ref(usd, noisy, t, ctx.float(), mmfs_features=[f.float() for f in feats], mmfs_mask=mask,
                            mmfs_module=hook, attention_head_dim=(2, 4))
    return dict(loss=(pred - noise) ** 2, pred=pred, target=noise, latents=latents, timesteps=t)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_stable_diffusion_forward_matches_restatement(dtype):
    sd, image, ctx, feats, mask = _tiny_sd(dtype)
    img = image.to(DEV)
    keep = img.clone()
    with torch.no_grad():
        out = sd(img, ctx.to(DEV, dtype), return_outputs=True, mmfs_features=[f.to(DEV, dtype) for f in feats],
                 mmfs_mask=mask.to(DEV), generator=torch.Generator(device=DEV).manual_seed(21))
    assert torch.equal(img, keep)                                   # normalised out of place
    ref = _sd_forward_ref(sd, image, ctx.to(dtype), [f.to(dtype) for f in feats], mask, 21, dtype)
    assert torch.equal(out["timesteps"].cpu(), ref["timesteps"])
    assert torch.equal(out["target"].float().cpu(), ref["target"])
    assert out["loss"].dtype == torch.float32 and out["loss"].shape == (2, 4, 16, 16)
    assert torch.equal(out["loss"], F.mse_loss(out["pred"].float(), out["target"].float(), reduction="none"))
    if dtype == torch.float32:
        for k in ("latents", "pred", "loss"):
            err = (out[k].float().cpu() - ref[k]).abs().max()
            assert err <= 1e-3 * ref[k].abs().max(), (k, (err / ref[k].abs().max()).item())
    else:
        for k in ("latents", "pred"):
            rel_max, rel_rms = _rel(out[k], ref[k])
            print(f"StableDiffusion.forward bf16 {k} vs restatement: max {rel_max:.3e} of max|ref|, relative RMS {rel_rms:.3e}")
            assert rel_max <= 6e-2 and rel_rms <= 3e-2, (k, rel_max, rel_rms)


def _tiny_image_decoder(uncond_prob):
    from mm_interleaved_b200.mm_interleaved import ImageDecoder
    from tests.test_unet_oracle import _tiny
    unet, net, _, _, _, _ = _tiny()
    torch.manual_seed(2)
    dec = ImageDecoder(perceiver_config=dict(num_queries=7, hidden_size=96, encoder_hidden_size=64, num_hidden_layers=2,
                                             num_attention_heads=4, intermediate_size=192, cross_attention_frequency=1,
                                             qk_normalization=True),
                       seq_len=7, embed_dim=96, unet=unet, mmfs_module=net, image_size=128, uncond_prob=uncond_prob,
                       vae=dict(block_out_channels=(32, 32, 64, 64), layers_per_block=1, with_encoder=True))
    return dec.to(DEV).eval()


def _decoder_inputs(n=3):
    g = torch.Generator().manual_seed(31)
    images = torch.rand((n, 3, 128, 128), generator=g).to(DEV)
    ctx = torch.randn((n, 5, 64), generator=g).to(DEV)
    feats = [torch.randn((n, 1, 96, s, s), generator=g).to(DEV) for s in (16, 8, 4, 2)]
    return images, ctx, feats, torch.ones((n, 1), device=DEV)


def test_image_decoder_uncond_prob_one_uses_the_negative_prompt():
    dec = _tiny_image_decoder(uncond_prob=1.0)
    images, ctx, feats, mmask = _decoder_inputs()
    cmask = torch.ones((3, 5), dtype=torch.long, device=DEV)
    with torch.no_grad():
        got = dec(images, ctx, cmask, mmfs_features=feats, mmfs_mask=mmask, generator=torch.Generator(device=DEV).manual_seed(4))
        g = torch.Generator(device=DEV).manual_seed(4)
        torch.rand((3, 1, 1), generator=g, device=DEV)              # the uncond draw comes first
        per = dec.decoder(images, dec.neg_prompt_embeds.expand(3, -1, -1), mmfs_features=feats, mmfs_mask=mmask, generator=g)
    assert got.dim() == 0
    assert torch.allclose(got, per.mean(), rtol=1e-6, atol=0), (got.item(), per.mean().item())


def test_image_decoder_masks_zero_images_but_keep_them_in_the_mean():
    dec = _tiny_image_decoder(uncond_prob=0.0)
    images, ctx, feats, mmask = _decoder_inputs()
    cmask = torch.ones((3, 5), dtype=torch.long, device=DEV)
    cmask[0, 2:] = 0                                                # image 0: <bos>, <soi> only -> not conditioned
    loss_mask = torch.tensor([1.0, 1.0, 0.0], device=DEV)           # image 2: masked by the caller
    with torch.no_grad():
        got = dec(images, ctx, cmask, image_loss_mask=loss_mask, mmfs_features=feats, mmfs_mask=mmask,
                  generator=torch.Generator(device=DEV).manual_seed(5))
        q = dec.perceiver_resampler(encoder_hidden_states=ctx, encoder_attention_mask=cmask)[0]
        per = dec.decoder(images, q, mmfs_features=feats, mmfs_mask=mmask, generator=torch.Generator(device=DEV).manual_seed(5))
    assert float(per[0].abs().sum()) > 0 and float(per[2].abs().sum()) > 0
    want = per[1].sum() / per.numel()
    assert torch.allclose(got, want, rtol=1e-5, atol=0), (got.item(), want.item())


def _mm_model(with_encoder):
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    from tests.golden.make_golden import LLAMA_TINY, seeded_state_dict
    from tests.test_mm_interleaved_gpu import N_TOK, ST
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(64, 128), layers_per_block=1, attention_head_dim=(2, 4),
                                        cross_attention_dim=96)
    net = m.MMFSNet(LLAMA_TINY["image_embed_dim"], (64, 128), 1, downsample_factor=2, spatial_shapes=[16, 8, 4, 2])
    vt_cfg = dict(clip_config=m.visual_tokenizer.CLIPVisionConfigLite(hidden_size=512, intermediate_size=512, num_hidden_layers=4,
                                                                     num_attention_heads=4, image_size=56, patch_size=14),
                  perceiver_config=dict(num_queries=N_TOK, hidden_size=192, encoder_hidden_size=512, cross_attention_frequency=2,
                                        num_hidden_layers=2, num_attention_heads=3, intermediate_size=384,
                                        qk_normalization=True), grid_size=4)
    img_cfg = dict(perceiver_config=dict(num_queries=7, hidden_size=96, encoder_hidden_size=LLAMA_TINY["hidden_size"],
                                         num_hidden_layers=2, num_attention_heads=4, intermediate_size=192,
                                         cross_attention_frequency=1, qk_normalization=True),
                   seq_len=7, embed_dim=96, unet=unet, mmfs_module=net, image_size=128, sd_base_seed=3,
                   vae=dict(block_out_channels=(32, 32, 64, 64), layers_per_block=1, with_encoder=with_encoder))
    model = m.MMInterleaved(llm_config=dict(LLAMA_TINY, vocab_size=62), txt_vocab_size=64, seq_len=32, special_token_dict=ST,
                            visual_tokenizer_config=vt_cfg, image_decoder_config=img_cfg,
                            image_embed_dim=LLAMA_TINY["image_embed_dim"], cross_attention_frequency=2,
                            spatial_shapes=LLAMA_TINY["spatial_shapes"])
    sd = model.state_dict()
    sd.update(seeded_state_dict({k: v for k, v in sd.items() if k.split(".")[0] in ("mm_decoder", "text_decoder", "soi_token",
                                                                                   "context_feat_proj")}, seed=2024))
    model.load_state_dict(sd)
    return model.to(DEV).eval()


def test_mm_interleaved_forward_adds_the_image_loss():
    from mm_interleaved_b200.mm_interleaved import context_features_for_image_decoder, mmfs_features_for_image_decoder
    from tests.test_mm_interleaved_gpu import ST, _batch
    ids, images, nimg, mask = _batch()
    ids, images, nimg, mask = ids.to(DEV), images.to(DEV), nimg.to(DEV), mask.to(DEV)
    dec_images = torch.rand((3, 3, 128, 128), generator=torch.Generator().manual_seed(41)).to(DEV)
    batch = dict(text_ids=ids, image_tensors=images, image_tensors_dec=dec_images, num_image_per_seq=nimg, attention_mask=mask)

    model = _mm_model(with_encoder=True)
    with torch.no_grad():
        out = model(**batch, generator=torch.Generator(device=DEV).manual_seed(7))
        assert {"loss", "loss_txt", "loss_img", "text_logits"} <= set(out) and "multiscale_features" not in out
        # the same inputs through ImageDecoder.forward directly
        pre = model._prepare_mm_embeds(ids, images, nimg)
        hid = model.mm_decoder(inputs_embeds=pre["mm_embeds"], attention_mask=mask, vision_hidden_states=pre["mmfs_features_mm"],
                               cross_attention_mask=pre["cross_attention_mask"], use_cache=False, return_dict=True).last_hidden_state
        ms = pre["multiscale_features"]
        ctx, cmask = context_features_for_image_decoder(hid, ids, ST["soi_token_id"], model.context_feat_proj, model.seq_len,
                                                        ms[0].shape[0])
        mf, mm = mmfs_features_for_image_decoder(ms, ids, ST["soi_token_id"])
        want = model.image_decoder(dec_images, ctx, cmask, mmfs_features=mf, mmfs_mask=mm,
                                   generator=torch.Generator(device=DEV).manual_seed(7))
        weighted = model(**batch, loss_img_weight=2.5, generator=torch.Generator(device=DEV).manual_seed(7))
    assert float(out["loss_img"]) > 0
    assert torch.allclose(out["loss_img"], want, rtol=1e-5, atol=0), (out["loss_img"].item(), want.item())
    assert torch.allclose(out["loss"], out["loss_txt"] + 10.0 * out["loss_img"], rtol=2 ** -22, atol=0)
    assert torch.allclose(weighted["loss"], weighted["loss_txt"] + 2.5 * weighted["loss_img"], rtol=2 ** -22, atol=0)

    plain = _mm_model(with_encoder=False)                           # decoder-only VAE: today's output
    res = plain.load_state_dict(model.state_dict(), strict=False)   # the same weights, the encoder half left out
    assert res.missing_keys == [] and res.unexpected_keys
    assert all(k.startswith(("image_decoder.decoder.vae.encoder.", "image_decoder.decoder.vae.quant_conv."))
               for k in res.unexpected_keys)
    with torch.no_grad():
        base = plain(**batch)
    assert set(base) == {"loss", "loss_txt", "text_logits", "multiscale_features"}
    assert torch.equal(base["loss"], base["loss_txt"])
    assert torch.allclose(base["loss_txt"], out["loss_txt"], rtol=1e-6, atol=0)
