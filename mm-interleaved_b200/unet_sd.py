"""SD-2.1-base UNet denoise step with the MMFS conditioning hook, H100-native assembly.

The reference does not contain the UNet arithmetic: it monkey-patches diffusers 0.20.0's
``UNet2DConditionModel.forward`` (utils/monkey_patch/sd_unet_forward_monkey_patch.py:17-371) to take three
extra keyword arguments -- ``mmfs_features``, ``mmfs_mask``, ``mmfs_module`` -- and to call
``mmfs_module(sample, down_block_res_samples, mmfs_features, mmfs_mask)`` between the mid block and the up blocks
(:316-326).  diffusers is neither under /root/reference nor in this image, so this file restates the published
SD-2.1-base architecture (block_out_channels (320, 640, 1280, 1280), 2 res-layers per block, 5/10/20/20 heads of
64, cross-attention dim 1024, linear projections, GEGLU feed-forward, GroupNorm(32)) with diffusers' parameter
naming so that a reference checkpoint's ``unet.*`` keys map one-to-one, and keeps the patched forward's
signature.  **Parity is unpinned** (no reference-side test, golden vector or importable implementation exists
here); the block-level formulas are checked against plain PyTorch statements in tests/test_unet_gpu.py.

H100 side: every self- and cross-attention runs in this repo's wgmma kernel (T in {4096, 1024, 256, 64},
head size 64, kv = 77 for cross attention), the MMFS branch in the fused sampler (sd_mmfs.py), LayerNorms in the
warp-per-row kernel, and every 3x3 / 1x1 convolution with Cin % 64 == 0 and Cout % 160 == 0 (all but conv_in / conv_out
when the model is bf16/f16 and channels-last) in the implicit-GEMM wgmma kernel (csrc/conv_igemm_sm100.cu) with the
ResNet block's time-embedding add and residual add fused into its epilogue; GroupNorm(+SiLU) runs in an NHWC kernel
(csrc/groupnorm_nhwc_sm100.cu) because torch's CUDA group_norm returns NCHW and would force a layout round trip
around every convolution.

Training path (the image loss): the convolutions on the kernel, GroupNorms, GEGLUs, attentions and LayerNorms call
the entry points of autograd_ops.py, which take the autograd Functions when autograd records the call; their forwards
run the same kernels as the inference path and their backwards carry the gradient to the UNet's inputs -- the context,
the MMFS hook and what feeds them.  The UNet's own weights get no gradient here: ``UNet2DConditionModel.forward`` under
autograd raises while any of them requires grad.  Nearest upsampling, ``cat``, the linears and ``conv_in`` /
``conv_out`` (library convolutions) stay on PyTorch autograd.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch
import torch.nn.functional as F
from torch import nn

from . import autograd_ops, ops
from ._cache import WeightCache
from .msda import records

USE_CONV_KERNEL = True      # tests flip this to compare against the cuDNN path on the same weights


def has_trainable_weights(unet: nn.Module) -> bool:
    """Whether a UNet parameter requires grad: the UNet's weights have no backward here, so its forward under autograd
    (and ``MMInterleaved.forward`` with the image loss on) refuses to run then."""
    return any(p.requires_grad for p in unet.parameters())


def _gn(mod: nn.GroupNorm, x: torch.Tensor, silu: bool) -> torch.Tensor:
    """``silu(mod(x))`` / ``mod(x)`` kept in NHWC by this repo's kernel when x is channels-last on the GPU."""
    if USE_CONV_KERNEL and ops.group_norm_supported(x):
        return autograd_ops.group_norm_nhwc(x, mod.num_groups, mod.weight, mod.bias, mod.eps, silu=silu)
    h = mod(x)
    return F.silu(h) if silu else h


class Conv2d(nn.Conv2d):
    """``nn.Conv2d`` that keeps its filter in the layouts ``ops.conv2d`` (KHWC) and ``ops.conv2d_up2x`` (folded) read."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._derived = WeightCache()

    def weight_khwc(self) -> torch.Tensor:
        return self._derived.get(self.weight, lambda: self.weight.permute(0, 2, 3, 1).contiguous(), key="khwc")

    def weight_up2x(self) -> torch.Tensor:
        return self._derived.get(self.weight, lambda: ops.fold_up2x_weights(self.weight), key="up2x")

    def weight_dgrad_khwc(self) -> torch.Tensor:
        """The data gradient's filter of a stride-1 layer (``ops.dgrad_weights_khwc``)."""
        return self._derived.get(self.weight, lambda: ops.dgrad_weights_khwc(self.weight.detach()), key="dgrad_khwc")

    def weight_dgrad_down2x(self) -> torch.Tensor:
        """The data gradient's phase filters of a 3x3 / stride-2 layer (``ops.fold_dgrad_down2x_weights``)."""
        return self._derived.get(self.weight, lambda: ops.fold_dgrad_down2x_weights(self.weight.detach()), key="dgrad_down2x")

    def uses_kernel(self, x: torch.Tensor) -> bool:
        """Whether ``fused`` runs this layer on the wgmma implicit-GEMM kernel for input x."""
        return (USE_CONV_KERNEL and x.is_contiguous(memory_format=torch.channels_last)
                and ops.conv2d_supported(x, self.weight, self.stride[0], self.padding[0]))

    def fused(self, x: torch.Tensor, add_bc: Optional[torch.Tensor] = None,
              residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``self(x) [+ add_bc[:, :, None, None]] [+ residual]`` -- on the wgmma implicit-GEMM kernel when the layer
        qualifies (``uses_kernel``), else on the library convolution."""
        if self.uses_kernel(x):
            if residual is not None and not residual.is_contiguous(memory_format=torch.channels_last):
                residual = residual.contiguous(memory_format=torch.channels_last)
            return ops.conv2d(x, self.weight_khwc(), self.bias, self.stride[0], self.padding[0], add_bc=add_bc,
                              residual=residual)
        h = self(x)
        if add_bc is not None:
            h = h + add_bc[:, :, None, None]
        return h if residual is None else h + residual


def _conv(mod: Conv2d, x: torch.Tensor, add_bc: Optional[torch.Tensor] = None,
          residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``mod.fused(x, add_bc, residual)``; a layer on the kernel through ``autograd_ops.conv`` (under autograd: same
    forward, dx and d residual in the backward), any other on the library convolution and PyTorch autograd."""
    if mod.uses_kernel(x):
        return autograd_ops.conv(x, mod, add_bc, residual)
    return mod.fused(x, add_bc, residual)


def timestep_embedding(timesteps: torch.Tensor, dim: int, max_period: int = 10000) -> torch.Tensor:
    """diffusers ``Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0)``: [cos | sin] of t * 10000^(-i/half)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=timesteps.device) / half)
    args = timesteps[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels, time_embed_dim):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


class ResnetBlock2D(nn.Module):
    """diffusers ``ResnetBlock2D``; ``temb_channels=None`` (the VAE decoder) has no ``time_emb_proj`` and no temb."""

    def __init__(self, in_channels, out_channels, temb_channels=1280, groups=32, eps=1e-5):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = Conv2d(in_channels, out_channels, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels) if temb_channels is not None else None
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps)
        self.conv2 = Conv2d(out_channels, out_channels, 3, padding=1)
        self.conv_shortcut = Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None

    def forward(self, x, temb=None):
        add = self.time_emb_proj(F.silu(temb)) if self.time_emb_proj is not None else None
        h = _conv(self.conv1, _gn(self.norm1, x, True), add_bc=add)
        skip = x if self.conv_shortcut is None else _conv(self.conv_shortcut, x)
        return _conv(self.conv2, _gn(self.norm2, h, True), residual=skip)


class Attention(nn.Module):
    """diffusers ``Attention`` (to_q / to_k / to_v without bias, to_out.0 with bias); softmax(q k^T / sqrt(d)) v."""

    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64):
        super().__init__()
        inner = heads * dim_head
        self.heads, self.dim_head = heads, dim_head
        kv = cross_attention_dim or query_dim
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(kv, inner, bias=False)
        self.to_v = nn.Linear(kv, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])

    def forward(self, x, context=None):
        B, T, _ = x.shape
        ctx = x if context is None else context
        q = self.to_q(x).view(B, T, self.heads, self.dim_head)
        k = self.to_k(ctx).view(B, ctx.shape[1], self.heads, self.dim_head)
        v = self.to_v(ctx).view(B, ctx.shape[1], self.heads, self.dim_head)
        return self.to_out[0](autograd_ops.attention_general(q, k, v))


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        hg = self.proj(x)
        if hg.is_cuda and hg.dtype != torch.float64 and (hg.shape[-1] // 2 * hg.element_size()) % 16 == 0:
            return autograd_ops.geglu(hg)
        h, gate = hg.chunk(2, dim=-1)
        return h * F.gelu(gate)


class FeedForward(nn.Module):
    def __init__(self, dim, mult=4):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim)])

    def forward(self, x):
        return self.net[2](self.net[0](x))


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, dim_head, cross_attention_dim):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, heads, dim_head)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, cross_attention_dim, heads, dim_head)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)

    def forward(self, x, context):
        n1, n2, n3 = self.norm1, self.norm2, self.norm3
        x = x + self.attn1(autograd_ops.layernorm(x, n1.weight, n1.bias, n1.eps))
        x = x + self.attn2(autograd_ops.layernorm(x, n2.weight, n2.bias, n2.eps), context)
        return x + self.ff(autograd_ops.layernorm(x, n3.weight, n3.bias, n3.eps))


class Transformer2DModel(nn.Module):
    def __init__(self, heads, dim_head, in_channels, cross_attention_dim, groups=32):
        super().__init__()
        inner = heads * dim_head
        self.norm = nn.GroupNorm(groups, in_channels, eps=1e-6)
        self.proj_in = nn.Linear(in_channels, inner)                       # use_linear_projection=True (SD 2.x)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, dim_head, cross_attention_dim)])
        self.proj_out = nn.Linear(inner, in_channels)

    def forward(self, x, context):
        B, C, H, W = x.shape
        h = _gn(self.norm, x, False).permute(0, 2, 3, 1).reshape(B, H * W, C)
        h = self.proj_in(h)
        for blk in self.transformer_blocks:
            h = blk(h, context)
        h = self.proj_out(h).reshape(B, H, W, C).permute(0, 3, 1, 2)
        return h + x


class Downsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = Conv2d(channels, channels, 3, stride=2, padding=1)

    def forward(self, x):
        return _conv(self.conv, x)


class Upsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = Conv2d(channels, channels, 3, padding=1)

    def forward(self, x):
        return _conv(self.conv, F.interpolate(x, scale_factor=2.0, mode="nearest"))


class DownBlock(nn.Module):
    def __init__(self, cin, cout, temb, heads, cross_dim, with_attn, add_down, layers=2):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb) for i in range(layers)])
        self.attentions = nn.ModuleList([Transformer2DModel(heads, cout // heads, cout, cross_dim) for _ in range(layers)]) if with_attn else None
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_down else None

    def forward(self, x, temb, context):
        outs = ()
        for i, res in enumerate(self.resnets):
            x = res(x, temb)
            if self.attentions is not None:
                x = self.attentions[i](x, context)
            outs += (x,)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs += (x,)
        return x, outs


class MidBlock(nn.Module):
    def __init__(self, ch, temb, heads, cross_dim):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, temb), ResnetBlock2D(ch, ch, temb)])
        self.attentions = nn.ModuleList([Transformer2DModel(heads, ch // heads, ch, cross_dim)])

    def forward(self, x, temb, context):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, context)
        return self.resnets[1](x, temb)


class UpBlock(nn.Module):
    def __init__(self, cin, cout, prev, temb, heads, cross_dim, with_attn, add_up, layers=3):
        super().__init__()
        res = []
        for i in range(layers):
            skip = cin if i == layers - 1 else cout
            inp = prev if i == 0 else cout
            res.append(ResnetBlock2D(inp + skip, cout, temb))
        self.resnets = nn.ModuleList(res)
        self.attentions = nn.ModuleList([Transformer2DModel(heads, cout // heads, cout, cross_dim) for _ in range(layers)]) if with_attn else None
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_up else None

    def forward(self, x, res_samples, temb, context):
        for i, res in enumerate(self.resnets):
            x = res(torch.cat([x, res_samples.pop()], dim=1), temb)
            if self.attentions is not None:
                x = self.attentions[i](x, context)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class UNet2DConditionModel(nn.Module):
    """SD-2.1-base UNet with the reference's patched forward signature (sd_unet_forward_monkey_patch.py:17-34)."""

    def __init__(self, in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
                 attention_head_dim=(5, 10, 20, 20), cross_attention_dim=1024):
        super().__init__()
        ch = list(block_out_channels)
        temb = ch[0] * 4
        self.block_out_channels = ch
        self.conv_in = nn.Conv2d(in_channels, ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], temb)
        self.down_blocks = nn.ModuleList()
        cin = ch[0]
        for i, cout in enumerate(ch):
            last = i == len(ch) - 1
            self.down_blocks.append(DownBlock(cin, cout, temb, attention_head_dim[i], cross_attention_dim,
                                              with_attn=not last, add_down=not last, layers=layers_per_block))
            cin = cout
        self.mid_block = MidBlock(ch[-1], temb, attention_head_dim[-1], cross_attention_dim)
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(ch))
        rev_heads = list(reversed(attention_head_dim))
        prev = rev[0]
        for i, cout in enumerate(rev):
            cin_skip = rev[min(i + 1, len(ch) - 1)]
            self.up_blocks.append(UpBlock(cin_skip, cout, prev, temb, rev_heads[i], cross_attention_dim,
                                          with_attn=i != 0, add_up=i != len(ch) - 1, layers=layers_per_block + 1))
            prev = cout
        self.conv_norm_out = nn.GroupNorm(32, ch[0], eps=1e-5)
        self.conv_out = nn.Conv2d(ch[0], out_channels, 3, padding=1)

    def forward(self, sample, timestep, encoder_hidden_states, mmfs_features: Optional[List[torch.Tensor]] = None,
                mmfs_mask: Optional[torch.Tensor] = None, mmfs_module=None):
        """Under autograd the gradient reaches ``encoder_hidden_states``, the MMFS hook and ``mmfs_features``; the
        UNet's own weights must be frozen (``unet.requires_grad_(False)``)."""
        if torch.is_grad_enabled() and has_trainable_weights(self):
            raise RuntimeError("UNet2DConditionModel.forward under autograd: the UNet's own weights have no backward here "
                               "(the image loss trains what feeds the UNet: the context, the MMFS hook and the features); "
                               "freeze them with unet.requires_grad_(False), or run under torch.no_grad()")
        feats = mmfs_features if isinstance(mmfs_features, (list, tuple)) else ()
        if self.conv_in.weight.is_cuda and records(sample, encoder_hidden_states, *feats, mmfs_module):
            # fail before the forward, not in loss.backward()
            autograd_ops.check_training_dtype("UNet2DConditionModel.forward under autograd", self.conv_in.weight)
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], device=sample.device)
        t = timestep.reshape(-1).expand(sample.shape[0])
        emb = self.time_embedding(timestep_embedding(t, self.block_out_channels[0]).to(sample.dtype))
        sample = self.conv_in(sample)
        res = (sample,)
        for blk in self.down_blocks:
            sample, outs = blk(sample, emb, encoder_hidden_states)
            res += outs
        sample = self.mid_block(sample, emb, encoder_hidden_states)
        if mmfs_module is not None:                                      # the hook of :316-326
            sample, res = mmfs_module(sample, res, mmfs_features, mmfs_mask)
        res = list(res)
        for blk in self.up_blocks:
            sample = blk(sample, res, emb, encoder_hidden_states)
        return self.conv_out(_gn(self.conv_norm_out, sample, True))


class GraphedUNet:
    """One UNet evaluation captured in a CUDA graph and replayed for every denoise step -- of every loop of the same
    shape.

    An evaluation is ~1200 kernel launches; issued eagerly, part of the wall time of a step is launch gaps.  Capturing
    + instantiating the graph costs more than one 50-step loop saves, so the graph must outlive the loop: ``sample`` and ``timestep`` (per step) and the context, the
    mask and the MMFS image-side state (per loop) all live in static buffers.  ``load`` refills the per-loop ones --
    the image-side state through ``MMFSNet.prepare(features, out=...)``, i.e. recomputed eagerly into the storage the
    graph reads -- and ``__call__`` replays.  The returned tensor lives in the graph's memory pool: consume it before
    the next call."""

    def __init__(self, unet, sample, timestep, ctx, mmfs_features, mmfs_mask, mmfs_module):
        self.unet, self.mmfs_module = unet, mmfs_module
        self.sample = sample.clone()
        self.t = timestep.clone()
        self.ctx = ctx.clone()
        self.mask = mmfs_mask.clone() if mmfs_mask is not None else None
        self.prepared = None
        if mmfs_module is not None and mmfs_features is not None:
            prep = getattr(mmfs_module, "prepare", None)
            self.prepared = prep(mmfs_features) if prep is not None else mmfs_features      # plain callables: read in place
        kw = dict(mmfs_features=self.prepared, mmfs_mask=self.mask, mmfs_module=mmfs_module)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            unet(self.sample, self.t, self.ctx, **kw)                  # warm-up: weight-derived caches, library handles
        torch.cuda.current_stream().wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        before = ops.launch_counter[0]
        with torch.cuda.graph(self.graph):
            self.out = unet(self.sample, self.t, self.ctx, **kw)
        self.launches = ops.launch_counter[0] - before                 # this repo's kernels inside one replay

    def load(self, ctx, mmfs_features, mmfs_mask):
        """New per-loop inputs (same shapes): context, mask and the MMFS image-side state."""
        self.ctx.copy_(ctx)
        if self.mask is not None:
            self.mask.copy_(mmfs_mask)
        if self.prepared is not None and hasattr(self.mmfs_module, "prepare"):
            self.mmfs_module.prepare(mmfs_features, out=self.prepared)

    def __call__(self, sample, timestep):
        self.sample.copy_(sample)
        self.t.copy_(timestep)
        self.graph.replay()
        ops.launch_counter[0] += self.launches
        return self.out


@torch.no_grad()
def denoise_loop(unet, latents, cond, uncond, mmfs_features, mmfs_mask, mmfs_module, num_steps=50, guidance=7.5,
                 num_train_timesteps=1000, cuda_graph: Optional[bool] = None, scheduler=None, generator=None,
                 graph_cache: Optional[dict] = None):
    """Classifier-free-guidance denoise loop in the shape of the patched pipeline ``__call__``
    (utils/monkey_patch/sd_pipeline_monkey_patch.py:153-218: ``set_timesteps``; CFG duplicates the MMFS inputs; per step
    ``scale_model_input``, one UNet call on the 2B batch, ``uncond + g (text - uncond)``, ``scheduler.step``).
    ``scheduler``: any object with ``set_timesteps / scale_model_input / step`` (scheduler.py; a diffusers scheduler
    works too).  Default = the reference's choice, DDPM ancestral sampling on the SD-2.1-base schedule (sd.py:48-50),
    its noise drawn from ``generator``.  ``graph_cache`` (a dict the caller keeps, e.g. ``StableDiffusion``): replay the
    UNet evaluation from a CUDA graph captured once per input shape and kept across loops (``GraphedUNet``);
    ``cuda_graph=True`` without a cache captures one graph for this loop only (costs more than it saves, see below)."""
    from .scheduler import DDPMScheduler, SD21_BASE_SCHEDULER
    if scheduler is None:
        scheduler = DDPMScheduler(**dict(SD21_BASE_SCHEDULER, num_train_timesteps=num_train_timesteps))
    scheduler.set_timesteps(num_steps, device=latents.device)
    ts_dev = scheduler.timesteps
    ts_host = getattr(scheduler, "_host_timesteps", None)
    if ts_host is None:
        ts_host = [int(t) for t in ts_dev.tolist()]
    own_step = hasattr(scheduler, "_host_timesteps")          # this repo's schedulers return the tensor directly
    latents = latents * getattr(scheduler, "init_noise_sigma", 1.0)
    ctx = torch.cat([uncond, cond], 0)
    feats2 = [torch.cat([f, f], 0) for f in mmfs_features] if mmfs_features is not None else None
    mask2 = torch.cat([mmfs_mask, mmfs_mask], 0) if mmfs_mask is not None else None
    if cuda_graph is None:
        # Capturing + instantiating the ~1200-node graph costs more than the launch overhead it removes from ONE
        # 50-step loop, so a graph is used only when the caller keeps it across loops (graph_cache), with the per-loop
        # MMFS state refreshed in place (GraphedUNet.load).
        cuda_graph = graph_cache is not None and latents.is_cuda
    runner = None
    if cuda_graph and graph_cache is not None:
        key = (tuple(latents.shape), latents.dtype, tuple(ctx.shape), id(unet), id(mmfs_module),
               None if feats2 is None else tuple(tuple(f.shape) for f in feats2), None if mask2 is None else tuple(mask2.shape))
        runner = graph_cache.get(key)
        if runner is not None:
            runner.load(ctx, feats2, mask2)
    for i, t_host in enumerate(ts_host):
        t = ts_dev[i]
        x2 = scheduler.scale_model_input(torch.cat([latents, latents], 0), t)
        if latents.is_cuda:
            x2 = x2.contiguous(memory_format=torch.channels_last)
        if cuda_graph:
            if runner is None:
                runner = GraphedUNet(unet, x2, t, ctx, feats2, mask2, mmfs_module)
                if graph_cache is not None:
                    graph_cache[key] = runner
            eps = runner(x2, t)
        else:
            eps = unet(x2, t, ctx, mmfs_features=feats2, mmfs_mask=mask2, mmfs_module=mmfs_module)
        e_u, e_c = eps.chunk(2)
        eps = e_u + guidance * (e_c - e_u)
        if own_step:
            latents = scheduler.step(eps, t_host, latents, generator=generator)
        else:                                                  # diffusers-style object
            latents = scheduler.step(eps, t, latents, generator=generator, return_dict=False)[0]
    return latents
