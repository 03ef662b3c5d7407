"""GPU parity of the implicit-GEMM wgmma convolution against F.conv2d in fp32 on the same bf16-rounded operands.
Tolerance: |err| <= 2e-2 * max|ref| (bf16 output rounding + fp32 accumulation order), mean |err| <= 2e-3 * max|ref|."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [
    # B, Cin, Cout, H, W, k, stride, pad, bias, add_bc, residual
    (2, 320, 320, 32, 32, 3, 1, 1, True, False, False),
    (2, 64, 160, 16, 16, 3, 1, 1, False, False, False),
    (2, 320, 320, 64, 64, 3, 2, 1, True, False, False),      # downsampler
    (2, 640, 320, 32, 32, 1, 1, 0, True, False, False),      # 1x1 shortcut
    (2, 1280, 1280, 8, 8, 3, 1, 1, True, True, True),        # 8x8 maps: tile spans two images; full ResNet-style epilogue
    (1, 960, 640, 32, 32, 3, 1, 1, True, True, False),       # up-block concat channels
    (2, 128, 160, 16, 32, 3, 1, 1, True, False, True),
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_conv_matches_torch(case, dtype):
    from mm_interleaved_b200 import ops
    B, Cin, Cout, H, W, k, stride, pad, has_bias, has_add, has_res = CASES[case]
    g = torch.Generator().manual_seed(case)
    x = torch.randn((B, Cin, H, W), generator=g).to(dtype)
    w = (torch.randn((Cout, Cin, k, k), generator=g) / (Cin * k * k) ** 0.5).to(dtype)
    bias = torch.randn(Cout, generator=g).to(dtype) if has_bias else None
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    add = torch.randn((B, Cout), generator=g).to(dtype) if has_add else None
    res = torch.randn((B, Cout, Ho, Wo), generator=g).to(dtype) if has_res else None
    xd = x.to(DEV).contiguous(memory_format=torch.channels_last)
    assert ops.conv2d_supported(xd, w, stride, pad)
    out = ops.conv2d(xd, w.permute(0, 2, 3, 1).contiguous().to(DEV), bias.to(DEV) if has_bias else None, stride, pad,
                     add_bc=add.to(DEV) if has_add else None,
                     residual=res.to(DEV).contiguous(memory_format=torch.channels_last) if has_res else None)
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.float(), w.float(), bias.float() if has_bias else None, stride, pad)
    if has_add:
        ref = ref + add.float()[:, :, None, None]
    if has_res:
        ref = ref + res.float()
    assert out.shape == ref.shape and out.is_contiguous(memory_format=torch.channels_last)
    err = (out.float().cpu() - ref).abs()
    assert err.max() <= 2e-2 * ref.abs().max(), (err.max().item(), ref.abs().max().item())
    assert err.mean() <= 2e-3 * ref.abs().max()


def test_unsupported_layers_are_reported():
    from mm_interleaved_b200 import ops
    x = torch.randn((2, 4, 64, 64), device=DEV, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    assert not ops.conv2d_supported(x, torch.empty(320, 4, 3, 3), 1, 1)          # conv_in: Cin = 4
    assert not ops.conv2d_supported(torch.empty((2, 320, 64, 64), device=DEV), torch.empty(320, 320, 3, 3), 1, 1)   # fp32


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.bfloat16, 1.6e-2), (torch.float16, 2e-3)])
@pytest.mark.parametrize("shape,silu", [((2, 320, 32, 32), True), ((3, 64, 16, 16), False), ((2, 960, 8, 8), True),
                                        ((1, 2560, 8, 8), True), ((2, 1920, 16, 16), False)])
def test_group_norm_nhwc_matches_torch(shape, silu, dtype, tol):
    """NHWC GroupNorm(32)(+SiLU) vs F.group_norm in fp32 on the same rounded inputs; |err| <= tol * max(1, |ref|)."""
    from mm_interleaved_b200 import ops
    g = torch.Generator().manual_seed(shape[1])
    x = (torch.randn(shape, generator=g) * 1.5 + 0.7).to(dtype)
    w = (1 + 0.2 * torch.randn(shape[1], generator=g)).to(dtype)
    b = (0.2 * torch.randn(shape[1], generator=g)).to(dtype)
    xd = x.to(DEV).contiguous(memory_format=torch.channels_last)
    out = ops.group_norm_nhwc(xd, 32, w.to(DEV), b.to(DEV), 1e-5, silu=silu)
    ref = torch.nn.functional.group_norm(x.float(), 32, w.float(), b.float(), 1e-5)
    if silu:
        ref = torch.nn.functional.silu(ref)
    assert out.is_contiguous(memory_format=torch.channels_last) and out.dtype == dtype
    err = (out.float().cpu() - ref).abs()
    assert (err <= tol * ref.abs().clamp_min(1.0)).all(), err.max().item()
