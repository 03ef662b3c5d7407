"""GPU tests of the image loss's backward through the frozen SD UNet: the two new kernels (GroupNorm-NHWC backward,
GEGLU backward), the convolution data gradient on the existing wgmma kernels, a (320, 640)-channel UNet with its MMFSNet
hook against float64 autograd through oracle/unet.py + oracle/sd_mmfs.py, and the model-level losses.

GroupNorm backward bound (elementwise; notation of tests/test_norm_kernels_gpu.py: u_T the element type's unit roundoff,
u = 2^-24, r = 1 / sqrt(var + eps), A = max |x| of the group).  The reference is float64 autograd of F.group_norm
(+ F.silu evaluated at the forward's rounding point round_T(z), what autograd of the 16-bit pipeline differentiates):
  * the kernel's xhat and r are fp32 statistics: xhat is off by S = c u (A r + |xhat|), r by c u A r relative (c = 16);
  * with SiLU, the kernel's rounded z can sit one ulp_T from round_T(z64) (its fp32 z errs by the forward's statistics
    term), which moves dz by at most |dy| / 2 times that (|silu''| <= 1/2): E_g = |gamma| |dy| (2 u_T |z| + S_z) / 2;
  * the fixed-order fp32 sums of g and g xhat over the group err by C_SUM u times the sums of magnitudes;
  * dx = r (g - mean g - xhat mean(g xhat)) carries these through, and is rounded once to T (u_T |ref|).
GEGLU backward: fp32 erff / expf within 2^-20 relative, one rounding: |err| <= u_T |ref| + 2^-18 (|dy v| + |dy g|)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
U = {F32: 2.0 ** -24, F16: 2.0 ** -11, BF16: 2.0 ** -8}
U32 = 2.0 ** -24
C_STAT, C_SUM = 16, 256
SUB = {t: U[t] * torch.finfo(t).smallest_normal for t in U}


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


@pytest.fixture
def strict_backends():
    """No TF32 in cuBLAS / cuDNN and deterministic cuDNN algorithms for one test; the previous flags come back after."""
    flags = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    try:
        yield
    finally:
        (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32,
         torch.backends.cudnn.deterministic) = flags


def _report(err, bound):
    i = int((err - bound).argmax())
    return f"max err {err.max().item():.3e}; worst excess at {i}: err {err.flatten()[i].item():.3e} > {bound.flatten()[i].item():.3e}"


# -------------------------------------------------------------------------------------------------- GroupNorm backward
def _gn_bwd_ref(x, dy, G, w, b, eps, silu):
    """float64 autograd on the device; returns (dx, bound) for the kernel's dtype."""
    dtype = x.dtype
    B, C = x.shape[:2]
    xd = x.double().requires_grad_(True)
    wd, bd = w.double(), b.double()
    z = F.group_norm(xd, G, wd, bd, eps)
    if silu:
        zr = z + (z.to(dtype).double() - z).detach()            # silu at the forward's rounded z, straight through
        y = F.silu(zr)
    else:
        y = z
    y.backward(dy.double())
    ref = xd.grad
    with torch.no_grad():
        xv = x.double()
        grp = xv.reshape(B, G, -1)
        mu, var, amax = grp.mean(-1), grp.var(-1, unbiased=False), grp.abs().amax(-1)
        r = torch.rsqrt(var + eps)
        pc = lambda t: t.repeat_interleave(C // G, dim=1)[:, :, None, None]
        xhat = (xv - pc(mu)) * pc(r)
        ar = pc(amax * r)
        gam, bet = wd.abs().view(1, C, 1, 1), bd.abs().view(1, C, 1, 1)
        S = C_STAT * U32 * (ar + xhat.abs())
        zz = z.detach()
        dyd = dy.double()
        if silu:
            s = torch.sigmoid(zz)
            dz = dyd * s * (1 + zz * (1 - s))
            Sz = S * gam + C_STAT * U32 * bet
            Eg = gam * dyd.abs() * (2 * U[dtype] * zz.abs() + Sz) / 2
        else:
            dz = dyd
            Eg = torch.zeros_like(dz)
        g = dz * wd.view(1, C, 1, 1)
        Eg = Eg + C_STAT * U32 * g.abs()
        gm = lambda t: pc(t.reshape(B, G, -1).mean(-1))         # group mean, broadcast back
        mgx = gm(g * xhat)
        inner = (Eg + gm(Eg) + xhat.abs() * gm(Eg * xhat.abs()) + S * mgx.abs() + xhat.abs() * gm(g.abs() * S)
                 + C_SUM * U32 * (gm(g.abs()) + xhat.abs() * gm((g * xhat).abs()))
                 + C_STAT * U32 * ar * (g.abs() + gm(g.abs()) + xhat.abs() * gm((g * xhat).abs())))
        bound = U[dtype] * ref.abs() + (1 + U[dtype]) * pc(r) * inner + SUB[dtype]
    return ref, bound


def _gn_bwd_case(x, G, eps, silu, seed):
    from mm_interleaved_b200 import ops
    g = _gen(seed)
    B, C = x.shape[:2]
    dtype = x.dtype
    w = (1 + 0.2 * torch.randn(C, generator=g)).to(dtype).to(DEV)
    b = (0.2 * torch.randn(C, generator=g)).to(dtype).to(DEV)
    dy = torch.randn(x.shape, generator=g).to(dtype).to(DEV).contiguous(memory_format=torch.channels_last)
    x = x.to(DEV).contiguous(memory_format=torch.channels_last)
    dx = ops.group_norm_nhwc_backward(x, dy, G, w, b, eps, silu=silu)
    again = ops.group_norm_nhwc_backward(x, dy, G, w, b, eps, silu=silu)
    assert dx.dtype == dtype and dx.shape == x.shape and dx.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(dx, again), "two runs of group_norm_nhwc_backward differ"
    ref, bound = _gn_bwd_ref(x, dy, G, w, b, eps, silu)
    err = (dx.double() - ref).abs()
    assert bool((err <= bound).all()), _report(err, bound)


# every (H = W, C) a GroupNorm of the SD-2.1 UNet sees (resnet norms, transformer norms, conv_norm_out)
UNET_GN_MAPS = [(64, 320), (64, 640), (64, 960), (32, 320), (32, 640), (32, 960), (32, 1280), (32, 1920),
                (16, 640), (16, 1280), (16, 1920), (16, 2560), (8, 1280), (8, 2560)]


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("hw,C", UNET_GN_MAPS)
def test_group_norm_backward_at_unet_maps(hw, C, dtype):
    g = _gen(hw * 7 + C)
    x = torch.randn(2, C, hw, hw, generator=g).to(dtype)
    _gn_bwd_case(x, 32, 1e-5, True, hw + C)
    _gn_bwd_case(x, 32, 1e-6, False, hw + C + 1)               # the transformer blocks' norm: eps 1e-6, no SiLU


@pytest.mark.parametrize("B,hw,C", [(16, 64, 320), (1, 8, 2560), (3, 32, 640), (1, 33, 320)])
def test_group_norm_backward_batches_and_ragged_maps(B, hw, C):
    x = torch.randn(B, C, hw, hw + 1 if hw == 33 else hw, generator=_gen(B * hw)).to(BF16)
    _gn_bwd_case(x, 32, 1e-5, True, B + hw)


GN_CONDITIONING = [(F32, 0, 1.0), (F32, 16, 1.0), (F32, 256, 1.0), (F32, 4096, 1.0),
                   (F16, 0, 1.0), (F16, 16, 1.0), (F16, 256, 1.0),
                   (BF16, 0, 1.0), (BF16, 16, 0.5), (BF16, 128, 0.5)]


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("dtype,ratio,sigma", GN_CONDITIONING)
def test_group_norm_backward_at_offset_groups(dtype, ratio, sigma, silu):
    """Groups offset to mean / sigma up to 4096 (fp32), with a few +-1000 sigma outlier channels."""
    B, C, H, W, G = 2, 320, 32, 32, 32
    g = _gen(ratio * 7 + int(silu))
    sign = (torch.randint(0, 2, (B, G), generator=g).double() * 2 - 1).repeat_interleave(C // G, dim=1)[:, :, None, None]
    x = sign * ratio * sigma + sigma * torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    if dtype != BF16 or ratio == 0:
        x[:, 3, 5, 7] += 1000 * sigma                              # outlier entries of two channels
        x[:, 77, 1, 2] -= 1000 * sigma
    _gn_bwd_case(x.to(dtype), G, 1e-5, silu, ratio + 3)


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("dtype", [F32, F16, BF16])
def test_group_norm_backward_near_constant_and_constant_groups(dtype, eps):
    B, C, H, W, G = 2, 320, 16, 16, 32
    cg = C // G
    g = _gen(int(1e6 * eps))
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    mu0 = {F32: 8.0, F16: 2.0 ** -2, BF16: 2.0 ** -6}[dtype]
    for gi in range(8):
        n = cg * H * W
        if dtype == F32:
            v = mu0 + 1e-4 * torch.randn(B, n, generator=g, dtype=torch.float64)
        else:
            v = mu0 + mu0 * 2.0 * U[dtype] * torch.randint(-2, 3, (B, n), generator=g).double()
        x[:, gi * cg:(gi + 1) * cg] = v.view(B, cg, H, W)
        x[:, (8 + gi) * cg:(9 + gi) * cg] = float(gi) - 3.5
    for silu in (False, True):
        _gn_bwd_case(x.to(dtype), G, eps, silu, gi + int(silu))


def test_group_norm_function_forward_is_the_inference_kernel():
    from mm_interleaved_b200 import autograd_ops, ops
    x = torch.randn(2, 640, 16, 16, device=DEV).to(BF16).contiguous(memory_format=torch.channels_last)
    w, b = torch.randn(640, device=DEV).to(BF16), torch.randn(640, device=DEV).to(BF16)
    xg = x.clone().requires_grad_(True)
    y = autograd_ops.group_norm_nhwc(xg, 32, w, b, 1e-5, silu=True)
    with torch.no_grad():
        assert torch.equal(y, ops.group_norm_nhwc(x, 32, w, b, 1e-5, silu=True))
    dy = torch.randn_like(y)
    y.backward(dy)
    assert torch.equal(xg.grad, ops.group_norm_nhwc_backward(x, dy.contiguous(memory_format=torch.channels_last), 32, w,
                                                             b, 1e-5, silu=True))


# ------------------------------------------------------------------------------------------------------ GEGLU backward
@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("rows,inter", [(2 * 4096, 1280), (2 * 77, 5120), (5, 13)])
def test_geglu_backward_against_float64(rows, inter, dtype):
    """Through GEGLUFunction at the UNet's widths; inter = 13 (odd rows: the element-wise path) on the kernel directly,
    as the forward kernel needs 16-byte rows."""
    from mm_interleaved_b200 import autograd_ops, ops
    g = _gen(rows + inter)
    vg = (3 * torch.randn(rows, 2 * inter, generator=g)).to(dtype).to(DEV)
    dy = torch.randn(rows, inter, generator=g).to(dtype).to(DEV)
    if inter % 8 == 0:
        x = vg.clone().requires_grad_(True)
        autograd_ops.geglu(x).backward(dy)
        got = x.grad
    else:
        got = ops.geglu_backward(vg, dy)
    assert torch.equal(got, ops.geglu_backward(vg, dy))
    vd = vg.double().requires_grad_(True)
    v, gate = vd.chunk(2, dim=-1)
    (v * F.gelu(gate)).backward(dy.double())
    ref = vd.grad
    dyd, vv, gg = dy.double(), v.detach(), gate.detach()
    scale = torch.cat([(dyd * gg).abs(), (dyd * vv).abs() * (1 + gg.abs())], -1)
    bound = U[dtype] * ref.abs() + 2.0 ** -18 * scale + SUB[dtype]
    err = (got.double() - ref).abs()
    assert bool((err <= bound).all()), _report(err, bound)


# -------------------------------------------------------------------------------------------------- convolution dgrad
def _conv_layer(cin, cout, k, stride, dtype, seed):
    from mm_interleaved_b200 import unet_sd
    torch.manual_seed(seed)
    conv = unet_sd.Conv2d(cin, cout, k, stride=stride, padding=k // 2).to(DEV, dtype).requires_grad_(False)
    with torch.no_grad():
        conv.weight.normal_(0, 1.0 / math.sqrt(cin * k * k))
    return conv


def _dgrad_check(conv, x_shape, dtype, seed, expect_kernel):
    """ConvFunction's dx (and d residual) against float64 conv2d_input.  The derived filters are exact re-indexings of W
    and the kernels accumulate in fp32 and round once: |err| <= u_T |ref| + 2^-12 sum |W| |dy|.  cuDNN's fallback may
    round inside its algorithm: u_T |ref| + 4 u_T sum |W| |dy|."""
    from mm_interleaved_b200 import autograd_ops, ops
    g = _gen(seed)
    x = torch.randn(x_shape, generator=g).to(dtype).to(DEV).contiguous(memory_format=torch.channels_last)
    xg = x.clone().requires_grad_(True)
    with torch.no_grad():
        res = conv.fused(x)                                     # a residual of the output's shape
    rg = res.clone().requires_grad_(True)
    y = autograd_ops.conv(xg, conv, None, rg)
    with torch.no_grad():
        assert torch.equal(y, conv.fused(x, None, res)), "ConvFunction's forward differs from the inference path"
    dy = torch.randn(y.shape, generator=g).to(dtype).to(DEV).contiguous(memory_format=torch.channels_last)
    before = ops.launch_counter[0]
    y.backward(dy)
    assert (ops.launch_counter[0] > before) == expect_kernel
    assert torch.equal(rg.grad, dy)
    ref = torch.nn.grad.conv2d_input(x_shape, conv.weight.double(), dy.double(), stride=conv.stride, padding=conv.padding)
    mag = torch.nn.grad.conv2d_input(x_shape, conv.weight.double().abs(), dy.double().abs(), stride=conv.stride,
                                     padding=conv.padding)
    err = (xg.grad.double() - ref).abs()
    bound = U[dtype] * ref.abs() + (2.0 ** -12 if expect_kernel else 4 * U[dtype]) * mag + SUB[dtype]
    assert bool((err <= bound).all()), _report(err, bound)


# (B, Cin, Cout, H = W, K, stride) of every SD-2.1 UNet convolution class with a kernel forward
UNET_CONVS = [(2, 320, 320, 64, 3, 1), (2, 640, 320, 64, 3, 1), (2, 960, 320, 64, 3, 1), (2, 640, 320, 64, 1, 1),
              (2, 960, 320, 64, 1, 1), (2, 320, 320, 64, 3, 2), (2, 320, 640, 32, 3, 1), (2, 640, 640, 32, 3, 1),
              (2, 320, 640, 32, 1, 1), (2, 1920, 640, 32, 1, 1), (2, 1280, 640, 32, 3, 1), (2, 640, 640, 32, 3, 2),
              (2, 1280, 1280, 16, 3, 1), (2, 2560, 1280, 16, 3, 1), (2, 1920, 1280, 16, 1, 1), (2, 1280, 1280, 16, 3, 2),
              (2, 1280, 1280, 8, 3, 1), (2, 2560, 1280, 8, 1, 1), (1, 2560, 1280, 16, 3, 1)]


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("B,cin,cout,hw,k,stride", UNET_CONVS)
def test_conv_dgrad_at_unet_layers(B, cin, cout, hw, k, stride, dtype):
    conv = _conv_layer(cin, cout, k, stride, dtype, cin + cout + hw)
    _dgrad_check(conv, (B, cin, hw, hw), dtype, hw + k, expect_kernel=True)


def test_conv_dgrad_falls_back_where_the_kernels_do_not_apply():
    """conv_out (its dgrad has Cout = 320 but Cin = 4) and an 8x8 map with an odd batch go to cuDNN's conv2d_input; a
    layer whose forward is on the kernel but whose swapped channels are not (Cin 64 -> Cout 160) falls back too."""
    from mm_interleaved_b200 import autograd_ops, ops
    conv_out = _conv_layer(320, 4, 3, 1, BF16, 1)
    dy = torch.randn(1, 4, 32, 32, device=DEV).to(BF16)
    before = ops.launch_counter[0]
    dx = autograd_ops.conv_input_grad(conv_out, dy, (1, 320, 32, 32))
    assert ops.launch_counter[0] == before
    ref = torch.nn.grad.conv2d_input((1, 320, 32, 32), conv_out.weight.double(), dy.double(), padding=1)
    assert float((dx.double() - ref).abs().max()) <= 2e-2 * float(ref.abs().max())
    odd = _conv_layer(1280, 1280, 3, 2, BF16, 2)
    dy = torch.randn(3, 1280, 8, 8, device=DEV).to(BF16).contiguous(memory_format=torch.channels_last)
    before = ops.launch_counter[0]
    dx = autograd_ops.conv_input_grad(odd, dy, (3, 1280, 16, 16))
    assert ops.launch_counter[0] == before
    ref = torch.nn.grad.conv2d_input((3, 1280, 16, 16), odd.weight.double(), dy.double(), stride=2, padding=1)
    assert float((dx.double() - ref).abs().max()) <= 2e-2 * float(ref.abs().max())
    swapped = _conv_layer(64, 160, 3, 1, BF16, 3)
    _dgrad_check(swapped, (2, 64, 32, 32), BF16, 4, expect_kernel=False)


# ------------------------------------------------------------------------------------------- UNet + MMFSNet gradients
CTX_DIM, FEAT_DIM, LAT = 1024, 256, 32


def _small(dtype):
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(320, 640), layers_per_block=1, attention_head_dim=(5, 10),
                                        cross_attention_dim=CTX_DIM).eval()
    net = m.MMFSNet(FEAT_DIM, (320, 640), 1, downsample_factor=2, spatial_shapes=[16, 8, 4, 2]).eval()
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.05)                    # non-zero: the hook's parameters get gradients
            blk.conv.bias.normal_(0, 0.05)
            blk.mmfs.sampling_offsets.weight.normal_(0, 0.01)
        for p in unet.parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
    g = _gen(1)
    x = torch.randn((2, 4, LAT, LAT), generator=g)
    ctx = torch.randn((2, 77, CTX_DIM), generator=g)
    feats = [torch.randn((2, 1, FEAT_DIM, s, s), generator=g) for s in (16, 8, 4, 2)]
    proj = torch.randn((2, 4, LAT, LAT), generator=g)
    return unet.to(DEV, dtype).requires_grad_(False), net.to(DEV, dtype), x, ctx, feats, proj


def _ref64(unet, net, x, t, ctx, feats, proj):
    """float64 autograd through the oracle's block functions (unet_forward_ref's control flow without its fp32 casts)."""
    from oracle.sd_mmfs import mmfsnet_ref
    from oracle.unet import _conv, _count, _lin, resnet_ref, timesteps_ref, transformer2d_ref
    sd = {k: v.detach().double() for k, v in unet.state_dict().items()}
    trainable = {n for n, p in net.named_parameters() if p.requires_grad}
    nsd = {k: v.detach().double().requires_grad_(k in trainable) for k, v in net.state_dict().items()}
    ctx = ctx.double().to(DEV).requires_grad_(True)
    feats = [f.double().to(DEV).requires_grad_(True) for f in feats]
    heads = [5, 10]
    with torch.device(DEV):
        tt = t.to(DEV).reshape(-1).expand(x.shape[0])
        emb = _lin(sd, "time_embedding.linear_2", F.silu(_lin(sd, "time_embedding.linear_1",
                                                                timesteps_ref(tt, 320).double())))
        sample = _conv(sd, "conv_in", x.double().to(DEV))
        res = (sample,)
        for b in range(_count(sd, "", "down_blocks")):
            p = f"down_blocks.{b}"
            attn = _count(sd, p + ".", "attentions") > 0
            for i in range(_count(sd, p + ".", "resnets")):
                sample = resnet_ref(sd, f"{p}.resnets.{i}", sample, emb)
                if attn:
                    sample = transformer2d_ref(sd, f"{p}.attentions.{i}", sample, ctx, heads[b])
                res += (sample,)
            if _count(sd, p + ".", "downsamplers") > 0:
                sample = _conv(sd, f"{p}.downsamplers.0.conv", sample, stride=2, padding=1)
                res += (sample,)
        sample = resnet_ref(sd, "mid_block.resnets.0", sample, emb)
        sample = transformer2d_ref(sd, "mid_block.attentions.0", sample, ctx, heads[-1])
        sample = resnet_ref(sd, "mid_block.resnets.1", sample, emb)
        sample, res = mmfsnet_ref(nsd, sample, list(res), feats, torch.ones((2, 1)), downsample_factor=2, n_down=len(res))
        res = tuple(res)
        for b in range(_count(sd, "", "up_blocks")):
            p = f"up_blocks.{b}"
            n = _count(sd, p + ".", "resnets")
            skips, res = res[-n:], res[:-n]
            attn = _count(sd, p + ".", "attentions") > 0
            for i in range(n):
                sample = resnet_ref(sd, f"{p}.resnets.{i}", torch.cat([sample, skips[-1 - i]], dim=1), emb)
                if attn:
                    sample = transformer2d_ref(sd, f"{p}.attentions.{i}", sample, ctx, heads[::-1][b])
            if _count(sd, p + ".", "upsamplers") > 0:
                sample = _conv(sd, f"{p}.upsamplers.0.conv", F.interpolate(sample, scale_factor=2.0, mode="nearest"))
        sample = F.silu(F.group_norm(sample, 32, sd["conv_norm_out.weight"], sd["conv_norm_out.bias"], 1e-5))
        out = _conv(sd, "conv_out", sample)
    (out * proj.double().to(DEV)).sum().backward()
    grads = {"context": ctx.grad, **{f"features.{i}": f.grad for i, f in enumerate(feats)}}
    grads.update({f"mmfs.{k}": v.grad for k, v in nsd.items() if v.grad is not None})
    return out.detach(), grads


def _ours(unet, net, x, t, ctx, feats, proj, dtype):
    ctx = ctx.to(DEV, dtype).requires_grad_(True)
    feats = [f.to(DEV, dtype).requires_grad_(True) for f in feats]
    net.zero_grad(set_to_none=True)
    out = unet(x.to(DEV, dtype).contiguous(memory_format=torch.channels_last), t.to(DEV), ctx, mmfs_features=feats,
               mmfs_mask=torch.ones((2, 1), device=DEV), mmfs_module=net)
    (out.float() * proj.to(DEV)).sum().backward()
    grads = {"context": ctx.grad, **{f"features.{i}": f.grad for i, f in enumerate(feats)}}
    grads.update({f"mmfs.{n}": p.grad for n, p in net.named_parameters() if p.grad is not None})
    return out.detach(), grads


def _grad_class(name):
    """Consumers of the MSDA location gradient (which jumps at pixel boundaries) get their own class: the offset path's
    parameters and, in the MMFSNet-level test, the gradient at the hook's sample and skip inputs (the queries)."""
    if any(s in name for s in (".sampling_offsets.", ".dynamic_offset_mask.", ".query_relpos.", ".query_norm.",
                               "input_grad/sample", "input_grad/res")):
        return "location"
    return "most"


# per-tensor relative error bounds (bf16, fp16).  Measured on an H100 (median / largest): "most" (55 tensors) bf16
# 1.9e-2 / 4.5e-2, fp16 2.2e-3 / 6.8e-3; "location" (35 tensors) bf16 0.25 / 0.31, fp16 7.8e-2 / 9.6e-2
GRAD_BOUND = {"most": {BF16: 6e-2, F16: 1e-2}, "location": {BF16: 0.6, F16: 0.15}}


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_unet_with_mmfs_hook_gradients_against_float64_oracle(dtype, strict_backends):
    unet, net, x, ctx, feats, proj = _small(dtype)
    t = torch.tensor(421)
    out, got = _ours(unet, net, x, t, ctx, feats, proj, dtype)
    ref_out, ref = _ref64(unet, net, x, t, ctx, feats, proj)
    assert float((out.double() - ref_out).norm() / ref_out.norm()) < (2e-2 if dtype == BF16 else 3e-3)
    assert sorted(got) == sorted(ref), (sorted(set(got) ^ set(ref)))
    rel = {n: float((got[n].double() - ref[n]).norm() / ref[n].norm().clamp_min(1e-30)) for n in ref}
    by_class = {}
    for n, e in rel.items():
        by_class.setdefault(_grad_class(n), []).append(e)
    summary = {c: (sorted(v)[len(v) // 2], max(v), len(v)) for c, v in by_class.items()}
    print(f"\n{dtype} relative gradient errors by class (median, max, count): {summary}")
    bad = {n: e for n, e in rel.items() if e > GRAD_BOUND[_grad_class(n)][dtype]}
    assert not bad, f"above the bound: {bad}; summary {summary}"


def test_unet_forward_under_autograd_is_bit_identical_to_inference():
    """Without the hook every UNet layer runs the same kernels under autograd: bit-identical output.  With it, the MMFS
    blocks take MMFS.forward_differentiable (the sampler's front end in PyTorch, the gather in the MSDA kernel, output_proj
    and the 1x1 conv as two maps) instead of the fused sampler with the folded output weight: a bounded difference."""
    unet, net, x, ctx, feats, proj = _small(BF16)
    xin = x.to(DEV, BF16).contiguous(memory_format=torch.channels_last)
    c = ctx.to(DEV, BF16)
    f = [v.to(DEV, BF16) for v in feats]
    kw = dict(mmfs_features=f, mmfs_mask=torch.ones((2, 1), device=DEV), mmfs_module=net)
    t = torch.tensor(421, device=DEV)
    with torch.no_grad():
        want, want_hook = unet(xin, t, c), unet(xin, t, c, **kw)
    got = unet(xin, t, c.clone().requires_grad_(True))
    assert got.requires_grad and torch.equal(got.detach(), want)
    got_hook = unet(xin, t, c.clone().requires_grad_(True), **kw)
    rel = float((got_hook.detach().double() - want_hook.double()).norm() / want_hook.double().norm())
    assert got_hook.requires_grad and rel < 3e-2, rel


def test_unet_gradients_are_run_to_run_identical(strict_backends):
    unet, net, x, ctx, feats, proj = _small(BF16)
    t = torch.tensor(421)
    _, a = _ours(unet, net, x, t, ctx, feats, proj, BF16)
    _, b = _ours(unet, net, x, t, ctx, feats, proj, BF16)
    for n in a:
        assert torch.equal(a[n], b[n]), n


# ------------------------------------------------------------------------------- MMFSNet against the reference's own
# The fixture's size has downsample factor 8, so its scale ratios reach 64: an offset is multiplied by up to 64 before it
# becomes a location, and the 16-bit rounding of the offsets and locations (8 significand bits in bf16) moves a sampling
# point by a large fraction of a pixel.  The forward output itself is then ~8 % off in bf16, so the bounds here are wider
# than the SD-sized UNet test's; fp16 (11 bits) is the tighter check, and each class's median is held too.  Measured on
# an H100 (median / largest): "most" (59 tensors) bf16 7.8e-2 / 0.17, fp16 9.4e-3 / 2.5e-2; "location" (40) bf16
# 0.55 / 0.76, fp16 0.16 / 0.57 (the mid block's sampling_offsets.weight).
FIXTURE_BOUND = {"most": {BF16: 0.3, F16: 5e-2}, "location": {BF16: 0.9, F16: 0.75}}
FIXTURE_MEDIAN = {"most": {BF16: 0.15, F16: 2e-2}, "location": {BF16: 0.7, F16: 0.3}}

def test_mmfsnet_gradients_against_the_reference_fixture(strict_backends):
    """tests/golden/mmfsnet_grad_tiny.npz holds the reference MMFSNet's float64 gradients (make_mmfsnet_grad.py): the
    hook's output, input and parameter gradients on the same weights and inputs, bf16 and fp16, per-tensor relative
    error by class."""
    import os

    import numpy as np

    import mm_interleaved_b200 as m
    from tests.golden.make_golden import MMFSNET_TINY, mmfsnet_state_dict
    from tests.golden.make_mmfsnet_grad import input_names, mmfsnet_grad_inputs
    from tests.golden.make_qformer_grad import sample_index
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mmfsnet_grad_tiny.npz"))
    summary, bad = {}, {}
    for dtype in (BF16, F16):
        net = m.MMFSNet(**MMFSNET_TINY)
        sd = mmfsnet_state_dict(net.state_dict())
        assert abs(float(sum(v.double().sum() for v in sd.values())) - float(z["checksum"])) < 1e-5
        net.load_state_dict(sd)
        net = net.to(DEV, dtype).eval()
        s, res, feats, mask, proj = mmfsnet_grad_inputs()
        inputs = [t.to(DEV, dtype).requires_grad_(True) for t in (s, *res, *feats)]
        out_s, out_res = net(inputs[0], inputs[1:1 + len(res)], inputs[1 + len(res):], mask.to(DEV))
        outs = [out_s, *out_res]
        sum((o.double() * p.to(DEV)).sum() for o, p in zip(outs, proj)).backward()
        got = {f"out/{i}": o.detach() for i, o in enumerate(outs)}
        got.update({f"input_grad/{n}": t.grad for n, t in zip(input_names(len(res), len(feats)), inputs)})
        got.update({f"grad/{n}": p.grad for n, p in net.named_parameters() if p.requires_grad})
        assert sorted(k for k in got if k.startswith("grad/")) == sorted(f"grad/{n}" for n in z["trainable"])
        rel = {}
        for k, t in got.items():
            ref = torch.from_numpy(z[k]).double()
            v = t.double().reshape(-1)[sample_index(t.numel()).to(DEV)].cpu()
            rel[k] = float((v - ref).norm() / ref.norm().clamp_min(1e-30))
        by = {}
        for k, e in rel.items():
            by.setdefault(_grad_class(k), []).append(e)
        summary[str(dtype)] = {c: (sorted(v)[len(v) // 2], max(v), len(v)) for c, v in by.items()}
        bad[dtype] = {k: e for k, e in rel.items() if e > FIXTURE_BOUND[_grad_class(k)][dtype]}
        bad[dtype].update({f"median of {c}": v[0] for c, v in summary[str(dtype)].items() if v[0] > FIXTURE_MEDIAN[c][dtype]})
    print(f"\nMMFSNet vs the reference fixture, relative errors by class (median, max, count): {summary}")
    assert not any(bad.values()), f"above the bound: {bad}"


# ------------------------------------------------------------------------------------------------- the model level
def _small_image_decoder(dtype):
    """An ImageDecoder with head dim 64 everywhere the backward kernels need it: UNet (128, 256) with 2 / 4 heads, a
    2-layer qk-norm Q-Former of hidden 128 over 2 heads, MMFSNet over 64-channel maps, the VAE encoder; 128^2 images.
    UNet and VAE frozen."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200 import unet_sd
    from mm_interleaved_b200.mm_interleaved import ImageDecoder
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(128, 256), layers_per_block=1, attention_head_dim=(2, 4),
                                        cross_attention_dim=128)
    net = m.MMFSNet(64, (128, 256), 1, downsample_factor=2, spatial_shapes=[16, 8, 4, 2])
    _liven_hook(net)
    dec = ImageDecoder(perceiver_config=dict(num_queries=7, hidden_size=128, encoder_hidden_size=64, num_hidden_layers=2,
                                             num_attention_heads=2, intermediate_size=256, cross_attention_frequency=1,
                                             qk_normalization=True),
                       seq_len=7, embed_dim=128, unet=unet, mmfs_module=net, image_size=128, uncond_prob=0.5,
                       vae=dict(block_out_channels=(32, 32, 64, 64), layers_per_block=1, with_encoder=True))
    dec = dec.to(DEV, dtype).eval()
    dec.decoder.unet.requires_grad_(False)
    dec.decoder.vae.requires_grad_(False)
    return dec


def _liven_hook(net):
    with torch.no_grad():
        for blk in list(net.mmfs_down_blocks) + [net.mmfs_mid_block]:
            blk.conv.weight.normal_(0, 0.05)                    # zero-initialised: would leave the hook without gradient


def _mixed_uncond_seed(n, p=0.5):
    """A generator seed whose first draw (ImageDecoder.forward's uncond draw) drops some prompts and keeps others."""
    for s in range(1000):
        u = torch.rand((n, 1, 1), generator=torch.Generator(device=DEV).manual_seed(s), device=DEV)
        if bool((u < p).any()) and bool((u >= p).any()):
            return s
    raise AssertionError("no seed found")


def test_image_decoder_backward_reaches_every_trainable_input_and_is_reproducible(strict_backends):
    dec = _small_image_decoder(BF16)
    g = torch.Generator().manual_seed(31)
    images = torch.rand((3, 3, 128, 128), generator=g).to(DEV)
    ctx = torch.randn((3, 5, 64), generator=g).to(DEV, BF16)
    feats = [torch.randn((3, 1, 64, s, s), generator=g).to(DEV, BF16) for s in (16, 8, 4, 2)]
    cmask = torch.ones((3, 5), dtype=torch.long, device=DEV)
    seed = _mixed_uncond_seed(3)

    def run():
        c = ctx.clone().requires_grad_(True)
        f = [t.clone().requires_grad_(True) for t in feats]
        dec.zero_grad(set_to_none=True)
        loss = dec(images, c, cmask, mmfs_features=f, mmfs_mask=torch.ones((3, 1), device=DEV),
                   generator=torch.Generator(device=DEV).manual_seed(seed))
        loss.backward()
        grads = {"context": c.grad, **{f"features.{i}": t.grad for i, t in enumerate(f)}}
        grads.update({n: p.grad for n, p in dec.named_parameters() if p.requires_grad})
        return loss.detach(), grads

    loss_a, a = run()
    loss_b, b = run()
    assert torch.equal(loss_a, loss_b)
    trainable = {n for n, p in dec.named_parameters() if p.requires_grad}
    assert "neg_prompt_embeds" in trainable and not any(n.startswith(("decoder.unet.", "decoder.vae.")) for n in trainable)
    for part in ("perceiver_resampler.", "neg_prompt_embeds", "decoder.mmfs_module.", "context", "features."):
        names = [n for n in a if n.startswith(part)]
        assert names and any(a[n] is not None and float(a[n].abs().max()) > 0 for n in names), part
    for n in a:
        assert (a[n] is None) == (b[n] is None), n
        if a[n] is not None:
            assert bool(torch.isfinite(a[n]).all()), n
            assert torch.equal(a[n], b[n]), n


def test_mm_interleaved_image_loss_backward_matches_the_module_level_computation(strict_backends):
    """One training step with the image loss on and the UNet frozen: ``MMInterleaved.forward(...)["loss"].backward()``
    against the same loss spelled out at module level -- gradients bit-identical, and present at the LLM's
    llama_cross_attn, context_feat_proj, neg_prompt_embeds, the image decoder's Q-Former and MMFSNet."""
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.mm_interleaved import context_features_for_image_decoder, mmfs_features_for_image_decoder
    from tests.golden.make_golden import LLAMA_TINY, seeded_state_dict
    from tests.test_mm_interleaved_gpu import N_TOK, ST, _batch
    from mm_interleaved_b200 import unet_sd
    torch.manual_seed(0)
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(128, 256), layers_per_block=1, attention_head_dim=(2, 4),
                                        cross_attention_dim=128)
    net = m.MMFSNet(LLAMA_TINY["image_embed_dim"], (128, 256), 1, downsample_factor=2, spatial_shapes=[16, 8, 4, 2])
    _liven_hook(net)
    vt_cfg = dict(clip_config=m.visual_tokenizer.CLIPVisionConfigLite(hidden_size=512, intermediate_size=512, num_hidden_layers=4,
                                                                     num_attention_heads=4, image_size=56, patch_size=14),
                  perceiver_config=dict(num_queries=N_TOK, hidden_size=192, encoder_hidden_size=512, cross_attention_frequency=2,
                                        num_hidden_layers=2, num_attention_heads=3, intermediate_size=384,
                                        qk_normalization=True), grid_size=4)
    img_cfg = dict(perceiver_config=dict(num_queries=7, hidden_size=128, encoder_hidden_size=LLAMA_TINY["hidden_size"],
                                         num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                                         cross_attention_frequency=1, qk_normalization=True),
                   seq_len=7, embed_dim=128, unet=unet, mmfs_module=net, image_size=128, sd_base_seed=3, uncond_prob=0.5,
                   vae=dict(block_out_channels=(32, 32, 64, 64), layers_per_block=1, with_encoder=True))
    model = m.MMInterleaved(llm_config=dict(LLAMA_TINY, vocab_size=62), txt_vocab_size=64, seq_len=32, special_token_dict=ST,
                            visual_tokenizer_config=vt_cfg, image_decoder_config=img_cfg,
                            image_embed_dim=LLAMA_TINY["image_embed_dim"], cross_attention_frequency=2,
                            spatial_shapes=LLAMA_TINY["spatial_shapes"])
    sd = model.state_dict()
    sd.update(seeded_state_dict({k: v for k, v in sd.items() if k.split(".")[0] in ("mm_decoder", "text_decoder", "soi_token",
                                                                                   "context_feat_proj")}, seed=2024))
    model.load_state_dict(sd)
    model = model.to(DEV, BF16).eval().freeze_like_reference()
    model.visual_tokenizer.requires_grad_(False)
    ids, images, nimg, mask = (t.to(DEV) for t in _batch())
    dec_images = torch.rand((3, 3, 128, 128), generator=torch.Generator().manual_seed(41)).to(DEV)
    batch = dict(text_ids=ids, image_tensors=images.to(BF16), image_tensors_dec=dec_images, num_image_per_seq=nimg,
                 attention_mask=mask)
    seed = _mixed_uncond_seed(3)
    with pytest.raises(RuntimeError, match=r"image-decoder loss has no backward here.*unet\.requires_grad_\(False\)"):
        model(**batch, generator=torch.Generator(device=DEV).manual_seed(seed))
    model.image_decoder.decoder.unet.requires_grad_(False)
    model.image_decoder.decoder.vae.requires_grad_(False)

    out = model(**batch, generator=torch.Generator(device=DEV).manual_seed(seed))
    out["loss"].backward()
    trainable = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    got = {n: p.grad.clone() for n, p in trainable if p.grad is not None}
    nonzero = lambda prefix: any(n.startswith(prefix) and float(g.abs().max()) > 0 for n, g in got.items())
    for prefix in ("mm_decoder.layers.0.llama_cross_attn.", "context_feat_proj.", "image_decoder.neg_prompt_embeds",
                   "image_decoder.perceiver_resampler.", "image_decoder.decoder.mmfs_module."):
        assert nonzero(prefix), prefix
    assert all(bool(torch.isfinite(g).all()) for g in got.values())
    model.zero_grad(set_to_none=True)

    # the same loss spelled out at module level
    pre = model._prepare_mm_embeds(ids, images.to(BF16), nimg)
    hid = model.mm_decoder(inputs_embeds=pre["mm_embeds"], attention_mask=mask, vision_hidden_states=pre["mmfs_features_mm"],
                           cross_attention_mask=pre["cross_attention_mask"], use_cache=False).last_hidden_state
    logits = model.text_decoder.logits(hid)
    gt = model._prepare_gt_text_ids(ids, mask, 0, None, None)
    loss_txt = F.cross_entropy(logits[:, :-1].float().transpose(1, 2), gt.contiguous())
    ms = pre["multiscale_features"]
    ctx, cmask = context_features_for_image_decoder(hid, ids, ST["soi_token_id"], model.context_feat_proj, model.seq_len,
                                                    ms[0].shape[0])
    mf, mm = mmfs_features_for_image_decoder(ms, ids, ST["soi_token_id"])
    loss_img = model.image_decoder(dec_images, ctx, cmask, mmfs_features=mf, mmfs_mask=mm,
                                   generator=torch.Generator(device=DEV).manual_seed(seed))
    loss = loss_txt * model.loss_txt_weight + loss_img * model.loss_img_weight
    assert torch.equal(loss.detach(), out["loss"].detach())
    loss.backward()
    for n, p in trainable:
        if n in got:
            assert torch.equal(p.grad, got[n]), n
        else:
            assert p.grad is None, n


def test_fp32_unet_under_autograd_fails_before_the_forward():
    from mm_interleaved_b200 import unet_sd
    unet = unet_sd.UNet2DConditionModel(block_out_channels=(128, 256), layers_per_block=1, attention_head_dim=(2, 4),
                                        cross_attention_dim=128).to(DEV).requires_grad_(False)
    x = torch.randn(1, 4, 16, 16, device=DEV).contiguous(memory_format=torch.channels_last)
    ctx = torch.randn(1, 7, 128, device=DEV, requires_grad=True)
    with pytest.raises(RuntimeError, match="bf16 / fp16 only"):
        unet(x, 1, ctx)
    with torch.no_grad():
        unet(x, 1, ctx)                                          # the inference path is unchanged
