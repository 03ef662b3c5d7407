"""GPU tests of the SD UNet assembly (parity unpinned: diffusers 0.20 is not available anywhere here).
The module is evaluated twice on the same weights: with this repo's kernels (attention, LayerNorm, fused MMFS
sampler) and with plain PyTorch statements of the same ops (softmax(QK^T/sqrt(d))V, F.layer_norm) patched in --
fp32, |err| <= 1e-3*|ref| + 1e-4*max|ref| -- and the MMFS hook must be called exactly once with 12 skip tensors
in the SD configuration."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _torch_attention(q, k, v, key_mask=None, causal=True, past=0, scale=None, force_generic=False):
    B, Tq, H, hd = q.shape
    s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * (scale or hd ** -0.5)
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v.float())
    return o.reshape(B, Tq, H * hd).to(q.dtype)


def _torch_layernorm(x, w, b, eps):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), w, b, eps)


def test_unet_kernels_vs_torch_statements_and_hook(monkeypatch):
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import ops, unet_sd
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(64, 128), layers_per_block=1, attention_head_dim=(2, 4),
                                        cross_attention_dim=96).to(DEV).eval()
    net = m.MMFSNet(96, (64, 128), 1, downsample_factor=2, spatial_shapes=[16, 8, 4, 2]).to(DEV).eval()
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.2)
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn((2, 4, 16, 16), device=DEV, generator=g)
    ctx = torch.randn((2, 7, 96), device=DEV, generator=g)
    feats = [torch.randn((2, 1, 96, s, s), device=DEV, generator=g) for s in (16, 8, 4, 2)]
    mask = torch.ones((2, 1), device=DEV)
    calls = []

    def hook(sample, res, f, mk):
        calls.append(len(res))
        return net(sample, res, f, mk)

    with torch.no_grad():
        got = unet(x, torch.tensor(500, device=DEV), ctx, mmfs_features=feats, mmfs_mask=mask, mmfs_module=hook)
        base = unet(x, torch.tensor(500, device=DEV), ctx)
        monkeypatch.setattr(ops, "attention", _torch_attention)
        monkeypatch.setattr(ops, "layernorm", _torch_layernorm)
        want = unet(x, torch.tensor(500, device=DEV), ctx, mmfs_features=feats, mmfs_mask=mask, mmfs_module=hook)
    assert got.shape == x.shape and calls == [4, 4]                  # conv_in + (res, down) + res = 4 skips in this tiny net
    assert (got - base).abs().max() > 1e-4                           # the MMFS branch really contributes
    err = (got - want).abs()
    assert (err <= 1e-3 * want.abs() + 1e-4 * want.abs().max()).all(), err.max()


def test_sd21_configuration_shapes_and_bf16_denoise_step():
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel().to(DEV, torch.bfloat16).eval().to(memory_format=torch.channels_last)
    net = m.MMFSNet(1024, (320, 640, 1280, 1280), 2).to(DEV, torch.bfloat16).eval()
    assert len(net.mmfs_down_blocks) == 12
    n_params = sum(p.numel() for p in unet.parameters())
    assert 8.5e8 < n_params < 8.8e8                                  # SD-2.1-base UNet: ~866 M parameters
    B = 1
    lat = torch.randn((B, 4, 64, 64), device=DEV, dtype=torch.bfloat16)
    cond = torch.randn((B, 77, 1024), device=DEV, dtype=torch.bfloat16) * 0.02
    feats = [torch.randn((B, 1, 1024, s, s), device=DEV, dtype=torch.bfloat16) for s in (64, 32, 16, 8)]
    out = unet_sd.denoise_loop(unet, lat, cond, torch.zeros_like(cond), feats, torch.ones((B, 1), device=DEV), net, num_steps=2)
    assert out.shape == lat.shape and torch.isfinite(out.float()).all()


def test_conv_kernel_path_matches_library_path_bf16():
    """Same bf16 weights, wgmma implicit-GEMM convolutions (fused temb / residual epilogues) vs the cuDNN path:
    |err| <= 3e-2 * max|ref| (bf16 rounding points differ: the fused epilogue rounds once instead of three times)."""
    from mm_interleaved_b200 import ops, unet_sd
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(320, 640), layers_per_block=1, attention_head_dim=(5, 10),
                                        cross_attention_dim=128).to(DEV, torch.bfloat16).eval().to(memory_format=torch.channels_last)
    x = torch.randn((2, 4, 32, 32), device=DEV, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    ctx = torch.randn((2, 7, 128), device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        n0 = ops.launch_counter[0]
        got = unet(x, torch.tensor(300, device=DEV), ctx)
        n_kernel = ops.launch_counter[0] - n0
        unet_sd.USE_CONV_KERNEL = False
        try:
            n0 = ops.launch_counter[0]
            want = unet(x, torch.tensor(300, device=DEV), ctx)
            n_lib = ops.launch_counter[0] - n0
        finally:
            unet_sd.USE_CONV_KERNEL = True
    assert n_kernel - n_lib >= 14                                    # the res-block / sampler convs really took the kernel path
    err = (got.float() - want.float()).abs()
    assert err.max() <= 3e-2 * want.float().abs().max(), (err.max().item(), want.float().abs().max().item())


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 5e-6), (torch.bfloat16, 8e-3), (torch.float16, 1e-3)])
def test_geglu_matches_torch(dtype, tol):
    """value * gelu(gate) on [value | gate] vs the torch statements of diffusers' GEGLU; |err| <= tol * max(1, |ref|)."""
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(3)
    x = (torch.randn((3, 37, 2 * 1280), generator=g) * 2).to(dtype)
    out = ops.geglu(x.to(DEV))
    h, gate = x.float().chunk(2, dim=-1)
    ref = h * torch.nn.functional.gelu(gate)
    err = (out.float().cpu() - ref).abs()
    assert out.shape == (3, 37, 1280) and (err <= tol * ref.abs().clamp_min(1.0)).all(), err.max().item()


def test_graphed_denoise_loop_matches_eager():
    """``denoise_loop(cuda_graph=True)`` (UNet evaluation captured once, replayed per step) gives the eager latents."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(320, 640), layers_per_block=1, attention_head_dim=(5, 10),
                                        cross_attention_dim=128).to(DEV, torch.bfloat16).eval().to(memory_format=torch.channels_last)
    net = m.MMFSNet(128, (320, 640), 1, downsample_factor=2, spatial_shapes=[32, 16, 8, 4]).to(DEV, torch.bfloat16).eval()
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.2)
    g = torch.Generator(device=DEV).manual_seed(2)
    lat = torch.randn((2, 4, 32, 32), device=DEV, dtype=torch.bfloat16, generator=g)
    cond = torch.randn((2, 7, 128), device=DEV, dtype=torch.bfloat16, generator=g)
    feats = [torch.randn((2, 1, 128, s, s), device=DEV, dtype=torch.bfloat16, generator=g) for s in (32, 16, 8, 4)]
    mask = torch.ones((2, 1), device=DEV)
    from mm_interleaved_b200.scheduler import DDIMScheduler      # deterministic update: the two runs must agree
    a = unet_sd.denoise_loop(unet, lat, cond, torch.zeros_like(cond), feats, mask, net, num_steps=4, cuda_graph=False,
                             scheduler=DDIMScheduler())
    b = unet_sd.denoise_loop(unet, lat, cond, torch.zeros_like(cond), feats, mask, net, num_steps=4, cuda_graph=True,
                             scheduler=DDIMScheduler())
    assert torch.isfinite(a.float()).all() and (a.float() - b.float()).abs().max() <= 1e-2 * a.float().abs().max()


def test_one_unet_graph_serves_loops_with_different_inputs():
    """A graph_cache makes ``denoise_loop`` capture the UNet evaluation once and REUSE it for later loops of the same shape:
    context, mask and the MMFS image-side state (MMFSNet.prepare(out=...)) are refreshed in place.  Two loops with different
    context / feature maps / latents through one cached graph must give the eager results of their own inputs -- a stale
    image-side buffer would reproduce the first loop's conditioning."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    from mm_interleaved_b200.scheduler import DDIMScheduler
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(320, 640), layers_per_block=1, attention_head_dim=(5, 10),
                                        cross_attention_dim=128).to(DEV, torch.bfloat16).eval().to(memory_format=torch.channels_last)
    net = m.MMFSNet(128, (320, 640), 1, downsample_factor=2, spatial_shapes=[32, 16, 8, 4]).to(DEV, torch.bfloat16).eval()
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.2)
    g = torch.Generator(device=DEV).manual_seed(3)
    mk = lambda: (torch.randn((2, 4, 32, 32), device=DEV, dtype=torch.bfloat16, generator=g),
                  torch.randn((2, 7, 128), device=DEV, dtype=torch.bfloat16, generator=g),
                  [torch.randn((2, 1, 128, s, s), device=DEV, dtype=torch.bfloat16, generator=g) for s in (32, 16, 8, 4)])
    sets = [mk(), mk()]
    mask = torch.ones((2, 1), device=DEV)
    cache = {}
    run = lambda st, gc: unet_sd.denoise_loop(unet, st[0], st[1], torch.zeros_like(st[1]), st[2], mask, net, num_steps=3,
                                              scheduler=DDIMScheduler(), graph_cache=gc).float().clone()
    eager = [run(st, None) for st in sets]
    graphed = [run(sets[0], cache), run(sets[1], cache), run(sets[0], cache)]
    assert len(cache) == 1                                   # one capture served all three loops
    scale = eager[0].abs().max()
    assert (eager[0] - eager[1]).abs().max() > 0.1 * scale   # the two input sets really differ
    for got, want in zip(graphed, (eager[0], eager[1], eager[0])):
        assert torch.isfinite(got).all() and (got - want).abs().max() <= 1e-2 * scale


def test_prepared_sd_features_equal_the_list_form():
    """MMFSNet with a PreparedSDFeatures (value_proj(LayerNorm(features)) computed once) = MMFSNet with the feature list."""
    import mm_interleaved_b200 as m
    torch.manual_seed(1)
    net = m.MMFSNet(128, (320, 640), 1, downsample_factor=2, spatial_shapes=[32, 16, 8, 4]).to(DEV, torch.bfloat16).eval()
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.2)
    g = torch.Generator(device=DEV).manual_seed(4)
    feats = [torch.randn((2, 1, 128, s, s), device=DEV, dtype=torch.bfloat16, generator=g) for s in (32, 16, 8, 4)]
    like = lambda blk, side: torch.randn((2, blk.query_norm.normalized_shape[0], side, side), device=DEV, dtype=torch.bfloat16,
                                         generator=g)               # a residual of the block's own width
    res = [like(blk, 16 if i < 2 else 8) for i, blk in enumerate(net.mmfs_down_blocks)]   # conv_in, layer | downsampler, layer
    sample = like(net.mmfs_mid_block, 8)
    mask = torch.ones((2, 1), device=DEV)
    with torch.no_grad():
        a_s, a_r = net(sample, res, feats, mask)
        pv = net.prepare(feats)
        b_s, b_r = net(sample, res, pv, mask)
        feats2 = [f * 0.5 + 1.0 for f in feats]
        net.prepare(feats2, out=pv)                              # refreshed in place: same storage, new conditioning
        c_s, _ = net(sample, res, pv, mask)
        d_s, _ = net(sample, res, feats2, mask)
    assert torch.equal(a_s, b_s) and all(torch.equal(x, y) for x, y in zip(a_r, b_r))
    assert torch.equal(c_s, d_s) and not torch.equal(c_s, a_s)
