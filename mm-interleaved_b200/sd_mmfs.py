"""``MMFSBlock`` / ``MMFSNet`` -- the MMFS conditioning branch of the SD-2.1 UNet, H100-native.

Mirrors ``mm_interleaved/models/decoders/sd_mmfs.py`` (MMFSBlock :44-145, MMFSNet :154-272): same
constructor arguments, parameter names (``mmfs_down_blocks.N.{query_norm,feat_norm,mmfs.*,pos_embed,conv}``,
``mmfs_mid_block.*``) and ``forward(sample, down_block_res_samples, mmfs_features, mmfs_mask)`` signature
(:230-236), so the patched UNet forward (utils/monkey_patch/sd_unet_forward_monkey_patch.py:316-326) can call it
unchanged.  Built for the denoise loop:

* ``LayerNorm(ms_feat)`` and ``value_proj`` run ONCE per conditioning tensor and are reused by every block call
  of every denoise step (the reference recomputes them 13 x steps x 2 times, SURVEY.md 8a a12);
* the zero-initialised 1x1 ``conv`` after MMFS is folded into ``output_proj`` (one GEMM instead of GEMM + conv);
* the per-pixel reference grid and the resized sin-cos position embedding are cached per query size;
* sampling runs in the fused MMFS kernel (pixel-grid reference points, 2-D image mask).

Under autograd (the image loss) a block runs ``_forward_differentiable`` instead: the LayerNorm Function on the
query and on the features (no feature cache), the frozen position embedding, ``MMFS.forward_differentiable`` on the
pixel grid, then ``output_proj`` and the 1x1 ``conv`` as two maps -- the folded weight is inference-only.
"""
from __future__ import annotations

import math
from functools import partial
from typing import List, Optional

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from ._cache import SourceCache, WeightCache
from .mmfs import MMFS


def sincos_pos_embed_2d(embed_dim: int, grid_size: int) -> torch.Tensor:
    """(grid_size^2, embed_dim) 2-D sine-cosine embedding: first half encodes the row index, second half the column
    index, each as [sin | cos] over 1/10000^(2i/d) frequencies (utils/pos_embed.py:45-95; float64 einsum like numpy)."""
    assert embed_dim % 4 == 0
    quarter = embed_dim // 4
    omega = 1.0 / 10000 ** (np.arange(quarter, dtype=np.float32) / np.float32(quarter))
    rows, cols = np.meshgrid(np.arange(grid_size, dtype=np.float32), np.arange(grid_size, dtype=np.float32), indexing="ij")

    def enc(pos):
        out = np.einsum("m,d->md", pos.reshape(-1), omega)
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)

    return torch.from_numpy(np.concatenate([enc(rows), enc(cols)], axis=1)).float()


def resize_abs_pos(abs_pos: torch.Tensor, tgt_len: int) -> torch.Tensor:
    """``get_abs_pos`` (utils/pos_embed.py:16-40) for embeddings without a cls token: bicubic resize of the square grid.
    The tables are frozen parameters, so callers cache the result on them (the reference re-interpolates per forward)."""
    src = int(math.sqrt(abs_pos.shape[0]))
    tgt = int(math.sqrt(tgt_len))
    if src == tgt:
        return abs_pos
    x = abs_pos.float().reshape(1, src, src, -1).permute(0, 3, 1, 2)
    x = F.interpolate(x, size=(tgt, tgt), mode="bicubic", align_corners=False)
    return x.permute(0, 2, 3, 1).flatten(0, 2).to(abs_pos.dtype)


def pixel_reference_points(h: int, w: int, device) -> torch.Tensor:
    """(1, h*w, 1, 2) pixel-centre grid x=(col+.5)/w, y=(row+.5)/h (sd_mmfs.py:15-28)."""
    ys = (torch.arange(h, device=device, dtype=torch.float32) + 0.5) / h
    xs = (torch.arange(w, device=device, dtype=torch.float32) + 0.5) / w
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    return torch.stack((gx.reshape(-1), gy.reshape(-1)), -1)[None, :, None, :].contiguous()


class MMFSBlock(nn.Module):
    def __init__(self, attn_dim=1024, query_dim=320, feat_dim=1024, num_heads=16, n_points=8, n_levels=1,
                 deform_ratio=1.0, norm_layer=partial(nn.LayerNorm, eps=1e-6), gradient_checkpointing=False,
                 grid_size=64, offset_init_magnitude=1, max_num_image_per_seq=10, spatial_shapes=[16],
                 base_spatial_shape=8, layer_idx=0):
        super().__init__()
        self.query_norm = norm_layer(query_dim)
        self.feat_norm = norm_layer(feat_dim)
        self.mmfs = MMFS(d_model=attn_dim, d_query=query_dim, d_value=feat_dim, d_out=query_dim, n_levels=n_levels,
                         n_heads=num_heads, n_points=n_points, ratio=deform_ratio,
                         offset_init_magnitude=offset_init_magnitude, spatial_shapes=spatial_shapes,
                         base_spatial_shape=base_spatial_shape, max_num_image_per_seq=max_num_image_per_seq,
                         layer_idx=layer_idx)
        self.pos_embed = nn.Parameter(sincos_pos_embed_2d(query_dim, grid_size), requires_grad=False)
        self.conv = nn.Conv2d(query_dim, query_dim, kernel_size=1, stride=1)
        nn.init.zeros_(self.conv.weight)       # zero_module (:148-151)
        nn.init.zeros_(self.conv.bias)
        self._geometry_cache = WeightCache()
        self._feat_cache = SourceCache()   # LayerNorm(ms_feat), identity-checked (see _cache.py)
        self._fused_out = WeightCache()

    def _reset_parameters(self):
        self.mmfs._reset_parameters()

    def _geometry(self, device, dtype, h, w, n_images, spatial_shapes):
        def build():
            ss = torch.tensor(list(spatial_shapes) * n_images, dtype=torch.long)
            starts = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
            pos = resize_abs_pos(self.pos_embed.detach(), h * w).to(device=device, dtype=dtype)
            return pixel_reference_points(h, w, device), ss.to(device), starts.to(device), pos
        key = (device, dtype, h, w, n_images, tuple(spatial_shapes))
        return self._geometry_cache.get(self.pos_embed, build, key)

    def _out_conv_fused(self):
        """conv1x1(output_proj(x)) = (Wc Wo) x + (Wc bo + bc): one GEMM."""
        ps = (self.mmfs.output_proj.weight, self.mmfs.output_proj.bias, self.conv.weight, self.conv.bias)

        def build():
            wc = self.conv.weight.view(self.conv.weight.shape[0], -1).float()
            w = (wc @ ps[0].float()).to(ps[0].dtype).contiguous()
            b = (wc @ ps[1].float() + ps[3].float()).to(ps[0].dtype).contiguous()
            return w, b
        return self._fused_out.get(ps, build)

    def normalised_features(self, ms_feat):
        n = self.feat_norm
        return self._feat_cache.get_or_build((ms_feat, n.weight, n.bias),
                                             lambda: ops.layernorm(ms_feat.contiguous(), n.weight, n.bias, n.eps),
                                             cache=not torch.is_grad_enabled())

    @torch.no_grad()
    def project_features(self, ms_feat):
        """value_proj(LayerNorm(ms_feat)) in the sampler's (B, N*HW, heads, D) layout: everything this block derives from
        the feature maps alone (constant over the denoise steps of a loop)."""
        n = self.feat_norm                      # no memoisation here: the caller owns the result (PreparedSDFeatures)
        return self.mmfs.project_value(ops.layernorm(ms_feat.contiguous(), n.weight, n.bias, n.eps), cache=False)

    def _records(self, sample, ms_feat) -> bool:
        return torch.is_grad_enabled() and (sample.requires_grad or (ms_feat is not None and ms_feat.requires_grad)
                                            or any(p.requires_grad for p in self.parameters()))

    def _forward_differentiable(self, sample, ms_feat, ms_feat_mask, spatial_shapes):
        from . import autograd_ops
        B, C, H, W = sample.shape
        n_images = ms_feat_mask.shape[-1]
        ref, ss, starts, pos = self._geometry(sample.device, sample.dtype, H, W, n_images, spatial_shapes)
        qn, fn = self.query_norm, self.feat_norm
        query = sample.flatten(2).transpose(1, 2).contiguous()                       # b c h w -> b (h w) c
        query = autograd_ops.layernorm(query, qn.weight, qn.bias, qn.eps) + pos
        feat = autograd_ops.layernorm(ms_feat.contiguous(), fn.weight, fn.bias, fn.eps)
        out = self.mmfs.forward_differentiable(query, ref, feat, ss, starts, ms_feat_mask)          # output_proj included
        out = F.linear(out, self.conv.weight.view(C, C), self.conv.bias)                          # the 1x1 conv, per token
        return out.transpose(1, 2).reshape(B, C, H, W)

    def forward(self, sample, ms_feat, ms_feat_mask, spatial_shapes, value=None):
        """sample (B, C_q, H, W); ms_feat (B, N, sum(H_l*W_l), C_v); ms_feat_mask (B, N); returns the residual (B, C_q, H, W).
        ``value`` (extension): ``project_features(ms_feat)`` computed by the caller (``ms_feat`` is then not read)."""
        if value is None and self._records(sample, ms_feat):
            return self._forward_differentiable(sample, ms_feat, ms_feat_mask, spatial_shapes)
        B, C, H, W = sample.shape
        n_images = ms_feat_mask.shape[-1]
        ref, ss, starts, pos = self._geometry(sample.device, sample.dtype, H, W, n_images, spatial_shapes)
        query = sample.flatten(2).transpose(1, 2).contiguous()                       # b c h w -> b (h w) c
        query = ops.layernorm(query, self.query_norm.weight, self.query_norm.bias, self.query_norm.eps) + pos
        feat = None if value is not None else self.normalised_features(ms_feat)
        # MMFS up to the sampled features, then output_proj and the 1x1 conv as one fused linear
        w, b = self._out_conv_fused()
        out = self.mmfs(query, ref, feat, ss, starts, input_padding_mask=None, attention_mask=ms_feat_mask,
                        output_weight=w, output_bias=b, value=value)
        return out.transpose(1, 2).reshape(B, C, H, W)


class PreparedSDFeatures:
    """Image-side state of the MMFSNet hook for ONE batch of context feature maps: per block,
    value_proj(LayerNorm(features)) -- what the blocks derive from the feature maps alone.  ``MMFSNet.prepare`` fills it
    once per denoise loop; passing it in place of the ``mmfs_features`` list makes the blocks read it instead of
    recomputing (or memoising by tensor identity).  With ``out=`` the values are written into existing storage: the
    static buffers a captured UNet graph reads (``unet_sd.GraphedUNet``)."""

    __slots__ = ("spatial_shapes", "values")

    def __init__(self, spatial_shapes, values):
        self.spatial_shapes = list(spatial_shapes)      # [(H_l, W_l)] of the feature maps
        self.values = list(values)                      # one per down block, then the mid block


class MMFSNet(nn.Module):
    def __init__(self, input_channel, block_out_channels, layers_per_block, downsample_factor=1, n_levels=4, n_points=8,
                 gradient_checkpointing=True, spatial_shapes=[64, 32, 16, 8]) -> None:
        super().__init__()
        self.downsample_factor = downsample_factor
        sd_shapes = [s // downsample_factor for s in spatial_shapes]

        def block(query_dim, shape_idx, layer_idx):
            return MMFSBlock(query_dim=query_dim, feat_dim=input_channel, n_points=n_points, n_levels=n_levels,
                             grid_size=64 // downsample_factor, spatial_shapes=spatial_shapes,
                             base_spatial_shape=sd_shapes[shape_idx], layer_idx=layer_idx)

        blocks = []
        blocks.append(block(block_out_channels[0], len(blocks) // 3, len(blocks)))          # conv_in skip (:190-197)
        for i, ch in enumerate(block_out_channels):
            for _ in range(layers_per_block):
                blocks.append(block(ch, len(blocks) // 3, len(blocks)))
            if i != len(block_out_channels) - 1:
                blocks.append(block(ch, len(blocks) // 3, len(blocks)))                    # downsampler skip
        self.mmfs_down_blocks = nn.ModuleList(blocks)
        self.mmfs_mid_block = block(block_out_channels[-1], -1, len(blocks))
        self._packed = SourceCache()       # the level-concatenated feature tensor, identity-checked (see _cache.py)

    @torch.no_grad()
    def prepare(self, mmfs_features: List[torch.Tensor], out: Optional[PreparedSDFeatures] = None) -> PreparedSDFeatures:
        """Run the feature-only part of every block once (see ``PreparedSDFeatures``)."""
        spatial_shapes = [(int(f.shape[-2]), int(f.shape[-1])) for f in mmfs_features]
        feats = torch.cat([f.flatten(3).transpose(2, 3) for f in mmfs_features], dim=2).contiguous()   # b n (h w) c
        blocks = list(self.mmfs_down_blocks) + [self.mmfs_mid_block]
        if out is None:
            return PreparedSDFeatures(spatial_shapes, [blk.project_features(feats) for blk in blocks])
        if out.spatial_shapes != spatial_shapes:
            raise ValueError("prepare(out=...): feature-map shapes differ from the prepared buffers")
        for dst, blk in zip(out.values, blocks):
            dst.copy_(blk.project_features(feats))
        return out

    def forward(self, sample: torch.Tensor, down_block_res_samples: List[torch.Tensor],
                mmfs_features, mmfs_mask: torch.Tensor):
        """``mmfs_features``: the list of feature maps (reference signature) or a ``PreparedSDFeatures`` (extension)."""
        assert len(down_block_res_samples) == len(self.mmfs_down_blocks)
        if isinstance(mmfs_features, PreparedSDFeatures):
            if torch.is_grad_enabled() and (any(t.requires_grad for t in (sample, *down_block_res_samples))
                                            or any(p.requires_grad for p in self.parameters())):
                raise RuntimeError("MMFSNet.forward under autograd: a PreparedSDFeatures was built under no_grad and "
                                   "would cut the gradient to the feature maps and the feature-side weights; pass the "
                                   "list of feature maps instead")
            pv = mmfs_features
            new_res = ()
            for res, blk, val in zip(down_block_res_samples, self.mmfs_down_blocks, pv.values):
                new_res += (res + blk(res, None, mmfs_mask, pv.spatial_shapes, value=val),)
            sample = sample + self.mmfs_mid_block(sample, None, mmfs_mask, pv.spatial_shapes, value=pv.values[-1])
            return sample, new_res
        spatial_shapes = [(int(f.shape[-2]), int(f.shape[-1])) for f in mmfs_features]
        # constant across the denoise steps of one loop: the same list of tensor objects comes back every step
        def pack():
            return torch.cat([f.flatten(3).transpose(2, 3) for f in mmfs_features], dim=2).contiguous()   # b n (h w) c
        feats = self._packed.get_or_build(list(mmfs_features), pack, cache=not torch.is_grad_enabled())
        new_res = ()
        for res, blk in zip(down_block_res_samples, self.mmfs_down_blocks):
            new_res += (res + blk(res, feats, mmfs_mask, spatial_shapes),)
        sample = sample + self.mmfs_mid_block(sample, feats, mmfs_mask, spatial_shapes)
        return sample, new_res
