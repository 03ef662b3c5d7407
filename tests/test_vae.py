"""CPU tests of the SD-2.1 VAE decoder (vae_sd.py) and of the fused upsample convolution's host side:

* the phase-form folding: ``fold_up2x_weights`` + four interleaved 2x2 convolutions equal
  ``conv3x3(interpolate(x, 2, "nearest"))`` in float64, at a non-square map, every border included;
* the decoder's state-dict keys follow diffusers' naming, a full VAE state dict loads with ``strict=False`` leaving
  only the encoder half unused, and the pre-rename attention names (query / key / value / proj_attn) load;
* ``mmfs_conv2d_up2x_nhwc`` validates its arguments before any CUDA call;
* a tiny fp32 ``AutoencoderKL`` equals the fp32 restatement in tests/vae_oracle.py."""
import pytest
import torch
import torch.nn.functional as F

from tests.vae_oracle import vae_decode_ref


def phase_conv_ref(x, w_phases):
    """conv3x3(up2x(x)) from folded weights: phase (py, px) = 2x2 conv over x padded by (1 - py, py) rows and
    (1 - px, px) columns, written to output pixels (2i + py, 2j + px)."""
    B, _, H, W = x.shape
    out = x.new_zeros((B, w_phases.shape[1], 2 * H, 2 * W))
    for py in range(2):
        for px in range(2):
            wf = w_phases[2 * py + px].permute(0, 3, 1, 2)            # (Cout, Cin, 2, 2)
            out[:, :, py::2, px::2] = F.conv2d(F.pad(x, (1 - px, px, 1 - py, py)), wf)
    return out


@pytest.mark.parametrize("H,W", [(5, 7), (1, 3), (6, 2)])
def test_fold_up2x_phase_convs_equal_interpolate_then_conv3x3(H, W):
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(H * 10 + W)
    x = torch.randn((2, 3, H, W), generator=g, dtype=torch.float64)
    w = torch.randn((4, 3, 3, 3), generator=g, dtype=torch.float64)
    wp = ops.fold_up2x_weights(w)
    assert wp.shape == (4, 4, 2, 2, 3) and wp.dtype == torch.float64
    ref = F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, padding=1)
    got = phase_conv_ref(x, wp)
    assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()


def test_fold_up2x_sums_in_fp32_and_rounds_once():
    from mm_interleaved_b200 import ops
    w = torch.randn((8, 64, 3, 3), generator=torch.Generator().manual_seed(1)).to(torch.bfloat16)
    wp = ops.fold_up2x_weights(w)
    assert wp.dtype == torch.bfloat16 and wp.is_contiguous()
    assert torch.equal(wp, ops.fold_up2x_weights(w.float()).to(torch.bfloat16))
    # phase (1, 1): taps {w0 + w1, w2} along both axes; tap (0, 0) sums the four weights of the top-left 2x2 block
    four = (w[:, :, 0, 0].float() + w[:, :, 0, 1].float() + w[:, :, 1, 0].float() + w[:, :, 1, 1].float()).to(torch.bfloat16)
    assert torch.equal(wp[3, :, 0, 0, :], four)
    assert torch.equal(wp[3, :, 1, 1, :], w[:, :, 2, 2])


def _expected_keys(chs=(128, 256, 512, 512), layers=2):
    keys = {"post_quant_conv.weight", "post_quant_conv.bias"}

    def add(p, *names):
        keys.update(f"{p}.{n}.{s}" for n in names for s in ("weight", "bias"))

    def resnet(p, cin, cout):
        add(p, "norm1", "conv1", "norm2", "conv2")
        if cin != cout:
            add(p, "conv_shortcut")

    add("decoder", "conv_in", "conv_norm_out", "conv_out")
    rev = list(reversed(chs))
    resnet("decoder.mid_block.resnets.0", rev[0], rev[0])
    resnet("decoder.mid_block.resnets.1", rev[0], rev[0])
    add("decoder.mid_block.attentions.0", "group_norm", "to_q", "to_k", "to_v", "to_out.0")
    prev = rev[0]
    for b, c in enumerate(rev):
        for i in range(layers + 1):
            resnet(f"decoder.up_blocks.{b}.resnets.{i}", prev if i == 0 else c, c)
        if b != len(rev) - 1:
            add(f"decoder.up_blocks.{b}.upsamplers.0", "conv")
        prev = c
    return keys


def test_state_dict_keys_follow_diffusers_naming():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    m = AutoencoderKL()
    sd = m.state_dict()
    assert set(sd) == _expected_keys()
    assert sum(v.numel() for v in sd.values()) == 49_490_199                     # 49.49 M, from the shapes
    assert sd["decoder.up_blocks.2.resnets.0.conv_shortcut.weight"].shape == (256, 512, 1, 1)
    assert sd["decoder.up_blocks.2.upsamplers.0.conv.weight"].shape == (256, 256, 3, 3)
    assert sd["decoder.conv_out.weight"].shape == (3, 128, 3, 3)


def test_full_vae_state_dict_and_deprecated_attention_names_load():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    src = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in src.parameters():
            p.copy_(torch.randn(p.shape, generator=g))
    sd = dict(src.state_dict())
    full = dict(sd, **{"encoder.conv_in.weight": torch.zeros(32, 3, 3, 3), "encoder.conv_in.bias": torch.zeros(32),
                       "quant_conv.weight": torch.zeros(8, 8, 1, 1), "quant_conv.bias": torch.zeros(8)})
    dst = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1)
    res = dst.load_state_dict(full, strict=False)
    assert res.missing_keys == [] and sorted(res.unexpected_keys) == sorted(
        ["encoder.conv_in.weight", "encoder.conv_in.bias", "quant_conv.weight", "quant_conv.bias"])
    old = {}
    renames = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "proj_attn"}
    for k, v in sd.items():
        for new, dep in renames.items():
            k = k.replace(f".attentions.0.{new}.", f".attentions.0.{dep}.")
        old[k] = v
    assert "decoder.mid_block.attentions.0.query.weight" in old and "decoder.mid_block.attentions.0.to_q.weight" not in old
    legacy = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1)
    legacy.load_state_dict(old)                                                     # strict: every key maps
    for k, v in legacy.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert "decoder.mid_block.attentions.0.query.weight" in old                   # the caller's dict is not renamed


def test_conv2d_up2x_argument_validation_without_gpu():
    from mm_interleaved_b200 import _lib
    lib = _lib.lib()
    rc = lib.mmfs_conv2d_up2x_nhwc(None, None, None, None, 2, 16, 16, 128, 128, _lib.BF16, None)
    assert rc == _lib.EINVAL and b"null pointer" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_up2x_nhwc(256, 256, None, 256, 0, 16, 16, 128, 128, _lib.BF16, None)
    assert rc == _lib.EINVAL and b"bad dimension" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_up2x_nhwc(256, 256, None, 256, 2, 16, 16, 128, 96, _lib.BF16, None)       # Cout % 128 != 0
    assert rc == _lib.EUNSUPPORTED and b"Cout % 128 == 0" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_up2x_nhwc(256, 256, None, 256, 2, 16, 16, 96, 128, _lib.BF16, None)       # Cin % 64 != 0
    assert rc == _lib.EUNSUPPORTED and b"Cin % 64 == 0" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_up2x_nhwc(256, 256, None, 256, 2, 12, 12, 128, 128, _lib.BF16, None)      # 12x12: no tiling
    assert rc == _lib.EUNSUPPORTED and b"tileable" in lib.mmfs_last_error()
    rc = lib.mmfs_conv2d_up2x_nhwc(256, 256, None, 256, 2, 16, 16, 128, 128, _lib.F32, None)
    assert rc == _lib.EUNSUPPORTED and b"bf16/f16" in lib.mmfs_last_error()


def test_tiny_fp32_vae_matches_oracle():
    from mm_interleaved_b200.vae_sd import AutoencoderKL
    torch.manual_seed(0)
    m = AutoencoderKL(block_out_channels=(32, 64, 64), layers_per_block=1).eval()
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "norm" in name:                                   # make the GroupNorm affine terms count
                p.add_(0.2 * torch.randn(p.shape, generator=g))
    z = torch.randn((2, 4, 6, 5), generator=g) * 3
    out = m.decode(z)
    ref = vae_decode_ref(m.state_dict(), z)
    assert out.shape == (2, 3, 24, 20) and out.dtype == torch.float32
    assert (out - ref).abs().max() <= 1e-5 * ref.abs().max()
