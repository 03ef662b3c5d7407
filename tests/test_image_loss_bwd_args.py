"""CPU tests of the image loss's training path: the argument checks of its two backward kernels
(``mmfs_groupnorm_nhwc_backward``, ``mmfs_geglu_backward``) and of their Python wrappers (every malformed or unsupported
call is rejected with MMFS_EINVAL / MMFS_EUNSUPPORTED and a message before any CUDA call), the two filter derivations of
the convolution data gradient in float64, and the guards that keep a frozen-UNet backward from dropping gradients."""
import pytest
import torch
import torch.nn.functional as F

GOOD = 0x1000            # stands for a valid device pointer; no call below gets far enough to dereference it
BF16, F16, F32, F64 = 2, 1, 0, 3


def _gn(**over):
    from mm_interleaved_b200 import _lib
    a = dict(x=GOOD, gamma=GOOD, beta=GOOD, dy=GOOD, dx=GOOD, scratch=GOOD, B=2, HW=64 * 64, C=320, G=32, eps=1e-5,
             silu=1, dtype=BF16)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_groupnorm_nhwc_backward(a["x"], a["gamma"], a["beta"], a["dy"], a["dx"], a["scratch"], a["B"], a["HW"],
                                          a["C"], a["G"], a["eps"], a["silu"], a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


def _geglu(**over):
    from mm_interleaved_b200 import _lib
    a = dict(vg=GOOD, dy=GOOD, dvg=GOOD, rows=2 * 4096, inter=1280, dtype=BF16)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_geglu_backward(a["vg"], a["dy"], a["dvg"], a["rows"], a["inter"], a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


@pytest.mark.parametrize("over,code,text", [
    (dict(x=None), "EINVAL", "null pointer"), (dict(dy=None), "EINVAL", "null pointer"),
    (dict(dx=None), "EINVAL", "null pointer"), (dict(scratch=None), "EINVAL", "null pointer"),
    (dict(B=0), "EINVAL", "bad sizes"), (dict(HW=0), "EINVAL", "bad sizes"), (dict(G=0), "EINVAL", "bad sizes"),
    (dict(G=30), "EINVAL", "bad sizes"), (dict(B=70000), "EINVAL", "bad sizes"),
    (dict(dtype=F64), "EUNSUPPORTED", "unsupported dtype"), (dict(dtype=7), "EUNSUPPORTED", "unsupported dtype"),
    (dict(C=324, G=4), "EUNSUPPORTED", "channel count"), (dict(C=4160, G=32), "EUNSUPPORTED", "8 KiB"),
    (dict(C=2560, dtype=F32), "EUNSUPPORTED", "8 KiB"),
    (dict(x=GOOD + 2), "EUNSUPPORTED", "aligned"), (dict(gamma=GOOD + 8), "EUNSUPPORTED", "aligned"),
])
def test_group_norm_backward_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _gn(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


@pytest.mark.parametrize("over,code,text", [
    (dict(vg=None), "EINVAL", "null pointer"), (dict(dy=None), "EINVAL", "null pointer"),
    (dict(dvg=None), "EINVAL", "null pointer"), (dict(rows=-1), "EINVAL", "bad shape"), (dict(inter=0), "EINVAL", "bad shape"),
    (dict(dtype=F32), "EUNSUPPORTED", "bf16"), (dict(dtype=F64), "EUNSUPPORTED", "bf16"), (dict(dtype=7), "EUNSUPPORTED", "bf16"),
])
def test_geglu_backward_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _geglu(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


def test_geglu_backward_empty_call_returns_before_the_pointers():
    from mm_interleaved_b200 import _lib
    assert _geglu(rows=0, vg=None)[0] == _lib.OK


def test_wrappers_refuse_bad_tensors():
    """Shapes, dtypes and devices are checked before the library sees the call (CPU tensors fail the first check)."""
    from mm_interleaved_b200 import ops
    with pytest.raises(RuntimeError, match="geglu_backward"):
        ops.geglu_backward(torch.zeros(4, 64), torch.zeros(4, 32))
    with pytest.raises(RuntimeError, match="group_norm_nhwc_backward"):
        ops.group_norm_nhwc_backward(torch.zeros(1, 64, 4, 4), torch.zeros(1, 64, 4, 4), 32)


def test_kernels_refuse_to_run_under_autograd():
    from mm_interleaved_b200 import ops
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.geglu_backward(torch.zeros(4, 64, requires_grad=True), torch.zeros(4, 32))
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.group_norm_nhwc_backward(torch.zeros(1, 64, 4, 4, requires_grad=True), torch.zeros(1, 64, 4, 4), 32)


def _up2x_phase_conv(x, phases):
    """``conv2d_up2x``'s arithmetic in float64: output (2i + py, 2j + px) = sum_{a, b} phases[p][:, a, b] x[i + a - 1 + py,
    j + b - 1 + px] over the zero-padded low-resolution input (phases (4, Cout, 2, 2, Cin))."""
    B, _, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    out = x.new_zeros(B, phases.shape[1], 2 * H, 2 * W)
    for py in range(2):
        for px in range(2):
            w = phases[2 * py + px].permute(0, 3, 1, 2)                 # (Cout, Cin, 2, 2)
            out[:, :, py::2, px::2] = F.conv2d(xp, w)[:, :, py:py + H, px:px + W]
    return out


def test_up2x_emulation_matches_the_forward_fold():
    """The emulation above is conv2d_up2x's contract: with fold_up2x_weights it equals conv3x3(nearest-2x(x))."""
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 6, 5, 4, generator=g, dtype=torch.float64)
    w = torch.randn(7, 6, 3, 3, generator=g, dtype=torch.float64)
    want = F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, padding=1)
    assert torch.allclose(_up2x_phase_conv(x, ops.fold_up2x_weights(w)), want, rtol=0, atol=1e-12)


@pytest.mark.parametrize("k,pad", [(3, 1), (1, 0)])
def test_dgrad_filter_of_stride_one_convolutions(k, pad):
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(k)
    w = torch.randn(12, 7, k, k, generator=g, dtype=torch.float64)
    dy = torch.randn(2, 12, 6, 5, generator=g, dtype=torch.float64)
    w_khwc = ops.dgrad_weights_khwc(w)
    assert tuple(w_khwc.shape) == (7, k, k, 12)
    got = F.conv2d(dy, w_khwc.permute(0, 3, 1, 2), padding=pad)             # the kernel's KHWC filter as OIHW
    want = torch.nn.grad.conv2d_input((2, 7, 6, 5), w, dy, padding=pad)
    assert float((got - want).abs().max()) <= 1e-12


def test_dgrad_phase_fold_of_stride_two_convolutions():
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(2)
    w = torch.randn(12, 7, 3, 3, generator=g, dtype=torch.float64)
    dy = torch.randn(2, 12, 4, 5, generator=g, dtype=torch.float64)
    phases = ops.fold_dgrad_down2x_weights(w)
    assert tuple(phases.shape) == (4, 7, 2, 2, 12)
    want = torch.nn.grad.conv2d_input((2, 7, 8, 10), w, dy, stride=2, padding=1)
    assert float((_up2x_phase_conv(dy, phases) - want).abs().max()) <= 1e-12
    wb = w.to(torch.bfloat16)                                  # each tap is one weight: the 16-bit fold is exact
    assert torch.equal(ops.fold_dgrad_down2x_weights(wb).double(), ops.fold_dgrad_down2x_weights(wb.double()))


def _tiny_unet():
    from mm_interleaved_b200 import unet_sd
    return unet_sd.UNet2DConditionModel(block_out_channels=(64, 128), layers_per_block=1, attention_head_dim=(2, 4),
                                        cross_attention_dim=96)


def test_trainable_unet_weights_raise_under_autograd():
    unet = _tiny_unet()
    x, ctx = torch.zeros(1, 4, 8, 8), torch.zeros(1, 7, 96, requires_grad=True)
    with pytest.raises(RuntimeError, match=r"unet\.requires_grad_\(False\)"):
        unet(x, 1, ctx)
    unet.conv_in.weight.requires_grad_(False)
    with pytest.raises(RuntimeError, match="UNet's own weights have no backward"):
        unet(x, 1, ctx)


def test_functions_refuse_trainable_weights():
    from mm_interleaved_b200 import autograd_ops, unet_sd
    conv = unet_sd.Conv2d(64, 160, 3, padding=1)
    with pytest.raises(RuntimeError, match="UNet's own weights have no backward"):
        autograd_ops.conv(torch.zeros(1, 64, 8, 8, requires_grad=True), conv)
    w = torch.ones(64, requires_grad=True)
    with pytest.raises(RuntimeError, match="UNet's own weights have no backward"):
        autograd_ops.group_norm_nhwc(torch.zeros(1, 64, 4, 4, requires_grad=True), 32, w, None)


def test_prepared_features_raise_under_autograd():
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.sd_mmfs import PreparedSDFeatures
    net = m.MMFSNet(96, (64, 128), 1, downsample_factor=2, spatial_shapes=[16, 8, 4, 2])
    res = [torch.zeros(1, 64, 8, 8)] * len(net.mmfs_down_blocks)
    prep = PreparedSDFeatures([(16, 16)], [None] * (len(net.mmfs_down_blocks) + 1))
    with pytest.raises(RuntimeError, match="PreparedSDFeatures was built under no_grad"):
        net(torch.zeros(1, 128, 4, 4), res, prep, torch.ones(1, 1))


def _mm_model(with_image_decoder):
    import mm_interleaved_b200 as m
    from tests.golden.make_golden import LLAMA_TINY
    vt_cfg = dict(clip_config=m.visual_tokenizer.CLIPVisionConfigLite(hidden_size=64, intermediate_size=64, num_hidden_layers=4,
                                                                     num_attention_heads=2, image_size=28, patch_size=14),
                  perceiver_config=dict(num_queries=2, hidden_size=64, encoder_hidden_size=64, cross_attention_frequency=2,
                                        num_hidden_layers=2, num_attention_heads=2, intermediate_size=64,
                                        qk_normalization=True), grid_size=2)
    st = dict(bos_token_id=1, eos_token_id=2, pad_token_id=0, soi_token_id=62, image_token_id=63)
    model = m.MMInterleaved(llm_config=dict(LLAMA_TINY, vocab_size=62), txt_vocab_size=64, seq_len=32, special_token_dict=st,
                            visual_tokenizer_config=vt_cfg, image_embed_dim=LLAMA_TINY["image_embed_dim"],
                            cross_attention_frequency=2, spatial_shapes=LLAMA_TINY["spatial_shapes"]).freeze_like_reference()
    model.visual_tokenizer.requires_grad_(False)
    if with_image_decoder:
        from mm_interleaved_b200.mm_interleaved import ImageDecoder
        model.image_decoder = ImageDecoder(perceiver_config=dict(num_queries=4, hidden_size=64, encoder_hidden_size=64,
                                                                 cross_attention_frequency=1, num_hidden_layers=1,
                                                                 num_attention_heads=2, intermediate_size=64),
                                           seq_len=4, embed_dim=64, unet=_tiny_unet(), mmfs_module=None, vae=False)
    model._has_image_loss = lambda: True
    return model


def test_mm_interleaved_image_loss_guard():
    """With the image loss on, autograd needs a UNet-backed image decoder whose UNet is frozen; the message names the
    recipe.  A frozen UNet passes the up-front check."""
    model = _mm_model(with_image_decoder=False)
    assert not model._image_loss_differentiable()
    ids = torch.ones(1, 4, dtype=torch.long)
    with pytest.raises(RuntimeError, match="the image-decoder loss has no backward here"):
        model(text_ids=ids, attention_mask=torch.ones_like(ids))
    model = _mm_model(with_image_decoder=True)
    assert not model._image_loss_differentiable()
    with pytest.raises(RuntimeError, match=r"the image-decoder loss has no backward here.*"
                                           r"model\.image_decoder\.decoder\.unet\.requires_grad_\(False\)"):
        model(text_ids=ids, attention_mask=torch.ones_like(ids))
    model.image_decoder.decoder.unet.requires_grad_(False)
    assert model._image_loss_differentiable()


def test_mmfsnet_trainable_set_matches_the_reference_fixture():
    """The reference's own MMFSNet decides which tensors train (tests/golden/mmfsnet_grad_tiny.npz); the names are this
    repository's too."""
    import os

    import numpy as np

    import mm_interleaved_b200 as m
    from tests.golden.make_golden import MMFSNET_TINY
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mmfsnet_grad_tiny.npz"))
    net = m.MMFSNet(**MMFSNET_TINY)
    assert sorted(n for n, p in net.named_parameters() if p.requires_grad) == [str(n) for n in z["trainable"]]


def test_mmfsnet_grad_generator_reproduces_the_fixture(tmp_path):
    import os

    import numpy as np

    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("the reference tree is not installed here")
    from tests.golden import make_mmfsnet_grad
    path = tmp_path / "mmfsnet_grad_tiny.npz"
    make_mmfsnet_grad.main(str(path))
    new = np.load(path)
    old = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mmfsnet_grad_tiny.npz"))
    assert sorted(new.files) == sorted(old.files)
    assert list(new["trainable"]) == list(old["trainable"])
    for k in new.files:
        if k.startswith(("grad/", "out/", "input_grad/")):
            np.testing.assert_allclose(new[k], old[k], rtol=1e-5, atol=1e-6 * float(np.abs(old[k]).max()), err_msg=k)
