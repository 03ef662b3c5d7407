"""The SD-UNet assembly (mm_interleaved_b200/unet_sd.py) and the denoise scheduler against INDEPENDENT restatements in
oracle/ (oracle/unet.py: state-dict-driven torch.nn.functional statement of diffusers 0.20's blocks following the
reference's patched forward, sd_unet_forward_monkey_patch.py:17-371; oracle/scheduler.py: DDPM eq. 6-7 in float64).
Still "parity unpinned" against diffusers itself (absent everywhere here) -- but no longer self-referential: a wrong
skip connection, time embedding, block order or scheduler coefficient in the product fails these tests.

Tolerances: fp32 tiny UNet (both the library-conv path and this repo's kernels) |err| <= 1e-3 |ref| + 1e-4 max|ref|;
full-width bf16 blocks max|err| <= 3e-2 max|ref| (bf16 storage at every layer boundary vs an fp32 oracle);
scheduler fp32 vs float64 oracle 2e-6 rel."""
import pytest
import torch

from oracle.scheduler import ddpm_step_ref, leading_timesteps, sd21_alphas_cumprod
from oracle.unet import resnet_ref, transformer2d_ref, unet_forward_ref


def test_ddpm_scheduler_matches_oracle_equations():
    from mm_interleaved_b200.scheduler import SD21_BASE_SCHEDULER, DDIMScheduler, DDPMScheduler
    for n in (30, 50):
        s = DDPMScheduler(**SD21_BASE_SCHEDULER)
        s.set_timesteps(n)
        assert s.timesteps.tolist() == leading_timesteps(n) and s._host_timesteps == leading_timesteps(n)
        assert torch.allclose(s.alphas_cumprod, sd21_alphas_cumprod(), rtol=0, atol=0)
        g = torch.Generator().manual_seed(n)
        x = torch.randn((2, 4, 8, 8), generator=g)
        for t in (s._host_timesteps[0], s._host_timesteps[n // 2], s._host_timesteps[-1]):
            eps, z = torch.randn(x.shape, generator=g), torch.randn(x.shape, generator=g)
            want = ddpm_step_ref(eps, t, x, z, n)
            got = s.step(eps, t, x, noise=z).double()
            assert float((got - want).abs().max()) <= 2e-6 * float(want.abs().max()), t
            assert s.scale_model_input(x, t) is x
        # seeded generator: reproducible draws, different from an explicit zero noise
        a = s.step(eps, 500 // (1000 // n) * (1000 // n) + 1, x, generator=torch.Generator().manual_seed(3))
        b = s.step(eps, 500 // (1000 // n) * (1000 // n) + 1, x, generator=torch.Generator().manual_seed(3))
        assert torch.equal(a, b)
    v = DDPMScheduler(**dict(SD21_BASE_SCHEDULER, prediction_type="v_prediction"))
    v.set_timesteps(30)
    t = v._host_timesteps[3]
    want = ddpm_step_ref(eps, t, x, z, 30, prediction_type="v_prediction")
    assert float((v.step(eps, t, x, noise=z).double() - want).abs().max()) <= 2e-6 * float(want.abs().max())
    d = DDIMScheduler()
    d.set_timesteps(4)
    assert d._host_timesteps == [999, 666, 333, 0]
    # eta = 0 DDIM: with a perfect epsilon the update lands on sqrt(a_prev) x0 + sqrt(1 - a_prev) eps
    acp = sd21_alphas_cumprod()
    x0 = torch.randn((1, 4, 4, 4), generator=g)
    e = torch.randn((1, 4, 4, 4), generator=g)
    xt = acp[666].sqrt() * x0 + (1 - acp[666]).sqrt() * e
    want = acp[333].sqrt() * x0 + (1 - acp[333]).sqrt() * e
    assert float((d.step(e, 666, xt) - want).abs().max()) < 1e-5


def _tiny():
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(64, 128), layers_per_block=1, attention_head_dim=(2, 4),
                                        cross_attention_dim=96).eval()
    net = m.MMFSNet(96, (64, 128), 1, downsample_factor=2, spatial_shapes=[16, 8, 4, 2]).eval()
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.2)
        for p in unet.parameters():                       # default inits are tiny for some blocks: make every path count
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, 4, 16, 16), generator=g)
    ctx = torch.randn((2, 7, 96), generator=g)
    feats = [torch.randn((2, 1, 96, s, s), generator=g) for s in (16, 8, 4, 2)]
    return unet, net, x, ctx, feats, torch.ones((2, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("use_kernels", [False, True])
def test_tiny_unet_with_mmfs_hook_matches_independent_oracle(use_kernels):
    from mm_interleaved_b200 import unet_sd
    from oracle.sd_mmfs import mmfsnet_ref
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    unet, net, x, ctx, feats, mask = _tiny()
    sd = {k: v.detach().clone() for k, v in unet.state_dict().items()}
    nsd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    oracle_hook = lambda s, res, f, mk: mmfsnet_ref(nsd, s, list(res), f, mk, downsample_factor=2, n_down=len(res))
    t = torch.tensor(421)
    want = unet_forward_ref(sd, x, t, ctx, mmfs_features=feats, mmfs_mask=mask, mmfs_module=oracle_hook, attention_head_dim=(2, 4))
    want_plain = unet_forward_ref(sd, x, t, ctx, attention_head_dim=(2, 4))
    assert float((want - want_plain).abs().max()) > 1e-3            # the hook is live in the oracle
    old = unet_sd.USE_CONV_KERNEL
    unet_sd.USE_CONV_KERNEL = use_kernels
    try:
        dev, dnet = unet.cuda(), net.cuda()
        xin = x.cuda().contiguous(memory_format=torch.channels_last) if use_kernels else x.cuda()
        with torch.no_grad():
            got = dev(xin, t.cuda(), ctx.cuda(), mmfs_features=[f.cuda() for f in feats], mmfs_mask=mask.cuda(), mmfs_module=dnet)
            got_plain = dev(xin, t.cuda(), ctx.cuda())
    finally:
        unet_sd.USE_CONV_KERNEL = old
    for g_, w_ in ((got, want), (got_plain, want_plain)):
        err = (g_.float().cpu() - w_).abs()
        assert bool((err <= 1e-3 * w_.abs() + 1e-4 * w_.abs().max()).all()), float(err.max())


@pytest.mark.gpu
def test_full_width_blocks_bf16_kernels_vs_oracle():
    """One SD-2.1-width ResNet block (320 -> 640 at 32x32, with the 1x1 shortcut and the time-embedding add) and one
    transformer block (5 heads x 64, 1024-wide context, T = 1024) on this repo's bf16 kernels (wgmma implicit-GEMM
    convolution, NHWC GroupNorm+SiLU, wgmma attention, LayerNorm, GEGLU) vs the fp32 oracle on the same weights."""
    from mm_interleaved_b200 import unet_sd
    torch.manual_seed(3)
    res = unet_sd.ResnetBlock2D(320, 640, 1280).eval()
    tr = unet_sd.Transformer2DModel(5, 64, 320, 1024).eval()
    with torch.no_grad():
        for mod in (res, tr):
            for p in mod.parameters():
                if p.dim() == 1:
                    p.add_(0.05 * torch.randn_like(p))
    g = torch.Generator().manual_seed(4)
    x = torch.randn((2, 320, 32, 32), generator=g)
    temb = torch.randn((2, 1280), generator=g)
    ctx = torch.randn((2, 77, 1024), generator=g)
    bf = lambda t: t.to(torch.bfloat16).float()
    rsd = {"r." + k: bf(v.detach()) for k, v in res.state_dict().items()}
    tsd = {"t." + k: bf(v.detach()) for k, v in tr.state_dict().items()}
    want_r = resnet_ref(rsd, "r", bf(x), bf(temb))
    want_t = transformer2d_ref(tsd, "t", bf(x), bf(ctx), heads=5)
    dt = torch.bfloat16
    with torch.no_grad():
        xin = x.cuda().to(dt).contiguous(memory_format=torch.channels_last)
        got_r = res.cuda().to(dt).to(memory_format=torch.channels_last)(xin, temb.cuda().to(dt))
        got_t = tr.cuda().to(dt)(xin, ctx.cuda().to(dt))
    for got, want in ((got_r, want_r), (got_t, want_t)):
        err = (got.float().cpu() - want).abs()
        assert float(err.max()) <= 3e-2 * float(want.abs().max()), (float(err.max()), float(want.abs().max()))
        assert float(err.mean()) <= 4e-3 * float(want.abs().max())


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_full_sd21_unet_with_mmfs_hook_bf16_vs_oracle():
    """The WHOLE SD-2.1 UNet (320 / 640 / 1280 / 1280 channels, 5 / 10 / 20 / 20 heads, 1024-wide context, 64 x 64 latents)
    with the full-size MMFSNet hook (4 feature maps 64 / 32 / 16 / 8 of one context image), one evaluation in bf16 on this
    repo's kernels against the fp32 oracle (oracle/unet.py + oracle/sd_mmfs.py) on the same bf16-rounded weights: the
    network of BASELINE cfg 4, every skip connection, down / up-sampler and attention head count included."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    from oracle.sd_mmfs import mmfsnet_ref
    torch.manual_seed(5)
    unet = unet_sd.UNet2DConditionModel().eval()
    net = m.MMFSNet(1024, (320, 640, 1280, 1280), 2, downsample_factor=1, spatial_shapes=[64, 32, 16, 8]).eval()
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.05)                  # zero-initialised in the reference: make the hook count
        for p_ in unet.parameters():
            if p_.dim() == 1:
                p_.add_(0.05 * torch.randn_like(p_))
    g = torch.Generator().manual_seed(6)
    x = torch.randn((1, 4, 64, 64), generator=g)
    ctx = torch.randn((1, 77, 1024), generator=g)
    feats = [torch.randn((1, 1, 1024, s_, s_), generator=g) for s_ in (64, 32, 16, 8)]
    mask = torch.ones((1, 1))
    bf = lambda t_: t_.to(torch.bfloat16).float()
    sd = {k: bf(v.detach()) for k, v in unet.state_dict().items()}
    nsd = {k: bf(v.detach()) for k, v in net.state_dict().items()}
    hook = lambda s_, res, f, mk: mmfsnet_ref(nsd, s_, list(res), f, mk, downsample_factor=1, n_down=len(res))
    t = torch.tensor(421)
    want = unet_forward_ref(sd, bf(x), t, bf(ctx), mmfs_features=[bf(f) for f in feats], mmfs_mask=mask, mmfs_module=hook)
    want_plain = unet_forward_ref(sd, bf(x), t, bf(ctx))
    assert float((want - want_plain).abs().max()) > 1e-2 * float(want.abs().max())      # the hook is live
    dt = torch.bfloat16
    dev = unet.cuda().to(dt).to(memory_format=torch.channels_last)
    dnet = net.cuda().to(dt)
    with torch.no_grad():
        got = dev(x.cuda().to(dt).contiguous(memory_format=torch.channels_last), t.cuda(), ctx.cuda().to(dt),
                  mmfs_features=[f.cuda().to(dt) for f in feats], mmfs_mask=mask.cuda(), mmfs_module=dnet)
    err = (got.float().cpu() - want).abs()
    scale = float(want.abs().max())
    assert torch.isfinite(got.float()).all()
    assert float(err.max()) <= 6e-2 * scale, (float(err.max()), scale)
    rel_rms = float(err.pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
    assert rel_rms <= 3e-2, rel_rms          # bf16 storage at ~60 layer boundaries against an fp32 oracle
