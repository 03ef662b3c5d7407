"""GPU tests of the SD-2.1 VAE decoder path (vae_sd.py) and its kernels (csrc/conv_igemm_sm100.cu).

Per-kernel bound, as in test_conv_gpu.py: max |err| <= 2e-2 * max|ref| and mean |err| <= 2e-3 * max|ref| against
fp32 on the same rounded operands (cuDNN with TF32 off).

The fused upsample convolution is also checked against fp32 ``conv3x3(interpolate(x))`` with the UNFOLDED weights.
The only extra difference there is the folded weights' rounding to 16 bit: each folded weight is one fp32 sum of
16-bit weights rounded once, so |wf16 - wf32| <= u |wf32| (u = 2^-8 for bf16, 2^-11 for f16).  The per-element bound
is therefore the kernel bound above plus u * (|x| conv |wf32|), computed with the same phase convolutions.

Whole decoder: the bound starts from the UNet's full-width bound (max <= 6e-2 of max|ref|, relative RMS <= 3e-2)."""
import pytest
import torch
import torch.nn.functional as F

from tests.test_vae import phase_conv_ref
from tests.vae_oracle import vae_decode_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}


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


CONV_CASES = [
    # B, Cin, Cout, H, W, k, residual   (Cout tile 128: Cout % 160 != 0)
    (2, 512, 512, 64, 64, 3, False),      # mid block / up block 0
    (1, 512, 256, 256, 256, 3, False),    # up block 2, first conv1
    (1, 512, 256, 256, 256, 1, False),    # its conv_shortcut
    (1, 256, 128, 512, 512, 3, True),     # up block 3: conv2 with the ResNet residual
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", range(len(CONV_CASES)))
def test_conv_cout_tile_128_at_vae_shapes(case, dtype):
    from mm_interleaved_b200 import ops
    B, Cin, Cout, H, W, k, has_res = CONV_CASES[case]
    g = torch.Generator(device=DEV).manual_seed(case)
    x = torch.randn((B, Cin, H, W), generator=g, device=DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    w = (torch.randn((Cout, Cin, k, k), generator=g, device=DEV) / (Cin * k * k) ** 0.5).to(dtype)
    bias = torch.randn(Cout, generator=g, device=DEV).to(dtype)
    res = torch.randn((B, Cout, H, W), generator=g, device=DEV).to(dtype).contiguous(memory_format=torch.channels_last) if has_res else None
    assert ops.conv2d_supported(x, w, 1, k // 2)
    out = ops.conv2d(x, w.permute(0, 2, 3, 1).contiguous(), bias, 1, k // 2, residual=res)
    ref = F.conv2d(x.float(), w.float(), bias.float(), 1, k // 2)
    if has_res:
        ref = ref + res.float()
    assert out.shape == ref.shape and out.is_contiguous(memory_format=torch.channels_last)
    _check(out, ref)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("Cin,Cout,H,W", [(128, 256, 16, 32), (256, 128, 24, 16), (64, 160, 8, 16)])
def test_conv2d_up2x_matches_phase_convs_and_interpolate_conv(Cin, Cout, H, W, dtype):
    from mm_interleaved_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(Cin + Cout + H)
    x = torch.randn((2, Cin, H, W), generator=g, device=DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    w = (torch.randn((Cout, Cin, 3, 3), generator=g, device=DEV) / (Cin * 9) ** 0.5).to(dtype)
    bias = torch.randn(Cout, generator=g, device=DEV).to(dtype)
    assert ops.conv2d_up2x_supported(x, w)
    wp = ops.fold_up2x_weights(w)
    out = ops.conv2d_up2x(x, wp, bias)
    assert out.shape == (2, Cout, 2 * H, 2 * W) and out.is_contiguous(memory_format=torch.channels_last)
    b = bias.float()[None, :, None, None]
    # (1) the kernel's arithmetic: the same folded, rounded weights in fp32
    _check(out, phase_conv_ref(x.float(), wp.float()) + b)
    # (2) the operation it replaces, with the unfolded weights
    ref = F.conv2d(F.interpolate(x.float(), scale_factor=2.0, mode="nearest"), w.float(), bias.float(), padding=1)
    fold_err = U[dtype] * phase_conv_ref(x.float().abs(), ops.fold_up2x_weights(w.float()).abs())
    err = (out.float() - ref).abs()
    assert (err <= 2e-2 * ref.abs().max() + fold_err).all(), (err - fold_err).max().item()


def _seeded_vae(**kw):
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    torch.manual_seed(0)
    m = AutoencoderKL(**kw).eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "norm" in name:                                    # make the GroupNorm affine terms count
                p.add_(0.2 * torch.randn(p.shape, generator=g))
    return m


def test_whole_decoder_sd21_widths_bf16_and_fp32_against_oracle():
    m = _seeded_vae().to(DEV)
    z = torch.randn((1, 4, 64, 64), generator=torch.Generator().manual_seed(2)) * 4
    sd = {k: v.to(DEV) for k, v in m.state_dict().items()}
    ref = vae_decode_ref(sd, z.to(DEV)).cpu()                      # fp32, TF32 off
    assert ref.shape == (1, 3, 512, 512)
    scale = ref.abs().max()

    f32 = m.decode(z.to(DEV)).cpu()
    assert f32.dtype == torch.float32
    assert (f32 - ref).abs().max() <= 1e-3 * scale, ((f32 - ref).abs().max() / scale).item()

    m16 = m.to(torch.bfloat16)
    a = m16.decode(z.to(DEV))
    b = m16.decode(z.to(DEV))
    assert a.dtype == torch.bfloat16 and torch.equal(a, b)        # fixed-order reductions: bit-identical
    err = a.float().cpu() - ref
    rel_max = (err.abs().max() / scale).item()
    rel_rms = (err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    print(f"whole decoder bf16 vs fp32 oracle: max {rel_max:.3e} of max|ref|, relative RMS {rel_rms:.3e}")
    assert rel_max <= 6e-2 and rel_rms <= 3e-2


def test_decoder_takes_the_kernels_in_16_bit():
    """The bf16 module runs its 3x3 / 1x1 convolutions and upsamplers in this repo's kernels (launch counter), and the
    cuDNN A/B path of the same module (unet_sd.USE_CONV_KERNEL = False) agrees with it."""
    from mm_interleaved_b200 import ops, unet_sd
    m = _seeded_vae(block_out_channels=(128, 256, 256), layers_per_block=1).to(DEV, torch.bfloat16)
    z = torch.randn((2, 4, 16, 32), generator=torch.Generator().manual_seed(3), device="cpu").to(DEV) * 4
    before = ops.launch_counter[0]
    own = m.decode(z)
    launches = ops.launch_counter[0] - before
    # 7 resnets (2 convs each) + 1 shortcut + 2 upsamplers; 8 GroupNorms (+ attention + conv_norm_out) x 2 kernels each
    assert launches >= 7 * 2 + 1 + 2
    unet_sd.USE_CONV_KERNEL = False
    try:
        lib = m.decode(z)
    finally:
        unet_sd.USE_CONV_KERNEL = True
    assert own.shape == lib.shape == (2, 3, 64, 128)
    err = (own.float() - lib.float()).abs()
    assert err.max() <= 6e-2 * lib.float().abs().max()


def test_generate_images_with_vae_returns_decoded_images():
    """MMInterleaved.generate(mode="generate_images") with a VAE in the image decoder: fp32 ``image`` (B, 3, 8h, 8w) in
    [0, 1], no ``latents`` key, equal to the oracle decode of the latents the same seeded call returns without a VAE."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    from tests.golden.make_golden import LLAMA_TINY, seeded_state_dict
    from tests.test_mm_interleaved_gpu import N_TOK, ST, _batch
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
                   vae=dict(block_out_channels=(128, 128, 256, 256), layers_per_block=1))
    model = m.MMInterleaved(llm_config=dict(LLAMA_TINY, vocab_size=62), txt_vocab_size=64, seq_len=32, special_token_dict=ST,
                            visual_tokenizer_config=vt_cfg, image_decoder_config=img_cfg,
                            image_embed_dim=LLAMA_TINY["image_embed_dim"], cross_attention_frequency=2,
                            spatial_shapes=LLAMA_TINY["spatial_shapes"])
    sd = model.state_dict()
    assert any(k.startswith("image_decoder.decoder.vae.decoder.") for k in sd)
    sd.update(seeded_state_dict({k: v for k, v in sd.items() if k.split(".")[0] in ("mm_decoder", "text_decoder", "soi_token",
                                                                                   "context_feat_proj")}, seed=2024))
    model.load_state_dict(sd)
    model = model.to(DEV).eval()
    vae = model.image_decoder.decoder.vae.to(torch.bfloat16)            # the VAE on the kernels, the rest fp32
    ids, images, nimg, mask = _batch()
    batch = dict(text_ids=ids.to(DEV), image_tensors=images.to(DEV), num_image_per_seq=nimg.to(DEV),
                 attention_mask=mask.to(DEV), meta=None)
    out = model.generate(mode="generate_images", **batch, num_inference_steps=3, guidance_scale=3.0)
    img = out["image"]
    assert "latents" not in out and img.dtype == torch.float32 and img.shape == (3, 3, 128, 128)
    assert float(img.min()) >= 0.0 and float(img.max()) <= 1.0

    model.image_decoder.decoder.vae_decode = None                       # same seeded call, latents out
    lat = model.generate(mode="generate_images", **batch, num_inference_steps=3, guidance_scale=3.0)["latents"]
    vsd = {k: v.float() for k, v in vae.state_dict().items()}
    ref = (vae_decode_ref(vsd, lat.float() / 0.18215) / 2 + 0.5).clamp(0, 1)
    err = (img - ref).float()
    scale = ref.abs().max()
    rel_max = (err.abs().max() / scale).item()
    rel_rms = (err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    print(f"generate_images with VAE vs oracle decode: max {rel_max:.3e} of max|ref|, relative RMS {rel_rms:.3e}")
    assert rel_max <= 6e-2 and rel_rms <= 3e-2
