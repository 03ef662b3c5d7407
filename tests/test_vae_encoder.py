"""CPU tests of the SD-2.1 VAE encoder (vae_sd.py), the posterior it returns, the scheduler's forward-diffusion
arithmetic (scheduler.py ``add_noise`` / ``get_velocity``) and the host side of the one-sided-pad downsample
convolution:

* ``with_encoder=True`` adds exactly diffusers' ``encoder.*`` / ``quant_conv.*`` keys (written out below) and
  34,163,664 parameters; a full VAE state dict, with the pre-rename attention names in the encoder's mid block, loads
  with ``strict=True``;
* a tiny fp32 ``encode`` equals the fp32 restatement in tests/image_loss_oracle.py;
* ``DiagonalGaussianDistribution``: the log-variance clamp at both ends, ``sample()`` and ``mode()``;
* ``add_noise`` / ``get_velocity`` against the float64 restatement, fp32 and bf16 samples, t = 0 and 999 included;
* ``mmfs_conv2d_down2x_nhwc`` validates its arguments before any CUDA call."""
import pytest
import torch

from tests.image_loss_oracle import add_noise_ref, get_velocity_ref, vae_encode_ref


def _encoder_keys(chs=(128, 256, 512, 512), layers=2):
    keys = {"quant_conv.weight", "quant_conv.bias"}

    def add(p, *names):
        keys.update(f"{p}.{n}.{s}" for n in names for s in ("weight", "bias"))

    def resnet(p, cin, cout):
        add(p, "norm1", "conv1", "norm2", "conv2")
        if cin != cout:
            add(p, "conv_shortcut")

    add("encoder", "conv_in", "conv_norm_out", "conv_out")
    prev = chs[0]
    for b, c in enumerate(chs):
        for i in range(layers):
            resnet(f"encoder.down_blocks.{b}.resnets.{i}", prev if i == 0 else c, c)
        if b != len(chs) - 1:
            add(f"encoder.down_blocks.{b}.downsamplers.0", "conv")
        prev = c
    resnet("encoder.mid_block.resnets.0", chs[-1], chs[-1])
    resnet("encoder.mid_block.resnets.1", chs[-1], chs[-1])
    add("encoder.mid_block.attentions.0", "group_norm", "to_q", "to_k", "to_v", "to_out.0")
    return keys


def test_encoder_keys_and_parameter_count_follow_diffusers():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    dec = AutoencoderKL().state_dict()
    full = AutoencoderKL(with_encoder=True).state_dict()
    assert set(full) - set(dec) == _encoder_keys() and set(dec) <= set(full)
    added = sum(full[k].numel() for k in set(full) - set(dec))
    assert added == 34_163_664                                                  # from diffusers' SD-2.1 shapes
    assert full["encoder.conv_in.weight"].shape == (128, 3, 3, 3)
    assert full["encoder.down_blocks.1.resnets.0.conv_shortcut.weight"].shape == (256, 128, 1, 1)
    assert full["encoder.down_blocks.2.downsamplers.0.conv.weight"].shape == (512, 512, 3, 3)
    assert full["encoder.conv_out.weight"].shape == (8, 512, 3, 3)
    assert full["quant_conv.weight"].shape == (8, 8, 1, 1)


def test_encoder_does_not_change_the_decoder_from_the_same_seed():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    torch.manual_seed(5)
    dec = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1).state_dict()
    torch.manual_seed(5)
    full = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1, with_encoder=True).state_dict()
    for k, v in dec.items():
        assert torch.equal(full[k], v), k


def test_full_vae_state_dict_with_deprecated_encoder_attention_names_loads_strictly():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    src = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1, with_encoder=True)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in src.parameters():
            p.copy_(torch.randn(p.shape, generator=g))
    sd = dict(src.state_dict())
    renames = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "proj_attn"}
    old = {}
    for k, v in sd.items():
        if k.startswith("encoder.mid_block.attentions.0."):
            for new, dep in renames.items():
                k = k.replace(f".attentions.0.{new}.", f".attentions.0.{dep}.")
        old[k] = v
    assert "encoder.mid_block.attentions.0.query.weight" in old and "decoder.mid_block.attentions.0.to_q.weight" in old
    dst = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1, with_encoder=True)
    dst.load_state_dict(old, strict=True)
    for k, v in dst.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_encode_without_encoder_raises():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    m = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1)
    assert m.encoder is None and m.quant_conv is None
    with pytest.raises(RuntimeError, match="no encoder"):
        m.encode(torch.zeros(1, 3, 16, 16))


def _tiny_vae():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    torch.manual_seed(0)
    m = AutoencoderKL(block_out_channels=(32, 64, 64), layers_per_block=1, with_encoder=True).eval()
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "norm" in name:                                   # make the GroupNorm affine terms count
                p.add_(0.2 * torch.randn(p.shape, generator=g))
    return m


def test_tiny_fp32_encode_matches_oracle():
    m = _tiny_vae()
    x = torch.rand((2, 3, 24, 20), generator=torch.Generator().manual_seed(6)) * 2 - 1
    post = m.encode(x).latent_dist
    mean, logvar = vae_encode_ref(m.state_dict(), x)
    assert post.mean.shape == (2, 4, 6, 5) and post.mean.dtype == torch.float32
    for got, ref in ((post.mean, mean), (post.logvar, logvar)):
        assert (got - ref).abs().max() <= 1e-5 * ref.abs().max()


def test_posterior_clamp_sample_and_mode():
    from mm_interleaved_b200.vae_sd import DiagonalGaussianDistribution
    moments = torch.randn((2, 8, 3, 5), generator=torch.Generator().manual_seed(7))
    moments[0, 4, 0, 0], moments[1, 7, 2, 4] = -45.0, 33.0                   # log-variance channels 4..7
    d = DiagonalGaussianDistribution(moments)
    assert torch.equal(d.mean, moments[:, :4])
    assert d.logvar[0, 0, 0, 0] == -30.0 and d.logvar[1, 3, 2, 4] == 20.0
    assert torch.equal(d.logvar.flatten()[1:-1], moments[:, 4:].flatten()[1:-1])
    assert torch.equal(d.std, torch.exp(0.5 * d.logvar))
    assert d.mode() is d.mean
    s = d.sample(torch.Generator().manual_seed(8))
    eps = torch.randn((2, 4, 3, 5), generator=torch.Generator().manual_seed(8))
    assert torch.equal(s, d.mean + d.std * eps)
    h = DiagonalGaussianDistribution(moments.to(torch.bfloat16)).sample(torch.Generator().manual_seed(8))
    assert h.dtype == torch.bfloat16 and h.shape == (2, 4, 3, 5)


@pytest.mark.parametrize("dtype,u", [(torch.float32, 2.0 ** -24), (torch.bfloat16, 2.0 ** -8)])
@pytest.mark.parametrize("pred", ["add_noise", "get_velocity"])
def test_add_noise_and_get_velocity_match_float64(dtype, u, pred):
    from mm_interleaved_b200.scheduler import DDPMScheduler, SD21_BASE_SCHEDULER
    sch = DDPMScheduler(**SD21_BASE_SCHEDULER)
    g = torch.Generator().manual_seed(9)
    x = torch.randn((5, 4, 8, 8), generator=g).to(dtype)
    n = torch.randn((5, 4, 8, 8), generator=g).to(dtype)
    t = torch.tensor([0, 999, 500, 1, 250])
    got = getattr(sch, pred)(x, n, t)
    assert got.dtype == dtype and got.shape == x.shape
    # diffusers moves alphas_cumprod to the sample's dtype first; the restatement gets the same rounded table
    acp = sch.alphas_cumprod.to(dtype)
    ref = (add_noise_ref if pred == "add_noise" else get_velocity_ref)(acp, x, n, t)
    a = acp.double()[t].view(-1, 1, 1, 1)
    first, second = (x, n) if pred == "add_noise" else (n, x)
    mag = a.sqrt() * first.double().abs() + (1 - a).sqrt() * second.double().abs()
    assert ((got.double() - ref).abs() <= 4 * u * mag + 1e-30).all()


def test_conv2d_down2x_argument_validation_without_gpu():
    from mm_interleaved_b200 import _lib
    lib = _lib.lib()
    rc = lib.mmfs_conv2d_down2x_nhwc(None, None, None, None, 2, 32, 32, 128, 128, _lib.BF16, None)
    assert rc == _lib.EINVAL and b"null pointer" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_down2x_nhwc(256, 256, None, 256, 0, 32, 32, 128, 128, _lib.BF16, None)
    assert rc == _lib.EINVAL and b"bad dimension" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_down2x_nhwc(256, 256, None, 256, 2, 32, -32, 128, 128, _lib.BF16, None)
    assert rc == _lib.EINVAL and b"bad dimension" in lib.mmfs_last_error()
    for H, W in ((31, 32), (32, 33)):
        rc = lib.mmfs_conv2d_down2x_nhwc(256, 256, None, 256, 2, H, W, 128, 128, _lib.BF16, None)
        assert rc == _lib.EINVAL and b"odd H or W" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_down2x_nhwc(256, 256, None, 256, 2, 32, 32, 128, 96, _lib.BF16, None)       # Cout % 128 != 0
    assert rc == _lib.EUNSUPPORTED and b"Cout % 128 == 0" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_down2x_nhwc(256, 256, None, 256, 2, 32, 32, 96, 128, _lib.BF16, None)       # Cin % 64 != 0
    assert rc == _lib.EUNSUPPORTED and b"Cin % 64 == 0" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_down2x_nhwc(256, 256, None, 256, 2, 24, 24, 128, 128, _lib.BF16, None)      # 12x12 out: no tiling
    assert rc == _lib.EUNSUPPORTED and b"tileable" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_down2x_nhwc(256, 256, None, 256, 1, 16, 16, 128, 128, _lib.BF16, None)      # 8x8 out, odd B
    assert rc == _lib.EUNSUPPORTED and b"tileable" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_down2x_nhwc(256, 256, None, 256, 2, 32, 32, 128, 128, _lib.F32, None)
    assert rc == _lib.EUNSUPPORTED and b"bf16/f16" in lib.mmfs_last_error()

