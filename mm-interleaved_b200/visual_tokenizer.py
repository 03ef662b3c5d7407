"""Visual tokenizer: CLIP ViT-L/14 + ViT-Adapter + Q-Former resampler, H100-native.

Mirrors the module tree / parameter names and the ``forward(image) -> {vis_embed, image_embeds,
multiscale_features}`` contract of the reference's
  encoders/visual_tokenizer.py:65-101          VisualTokenizer
  encoders/vit_adapter/vit_adapter_hf.py:42-167 CLIPVisionTransformerAdapter (CLIP ViT-L/14, 24 layers split 4 x 6)
  encoders/vit_adapter/adapter_modules.py       SpatialPriorModule :267-328, Injector / Extractor :92-154,
                                                ConvFFN / DWConv :52-89, InteractionBlockWithCls :198-233
  encoders/vit_adapter/ops/modules/ms_deform_attn.py:27-131  MSDeformAttn (classic single-image variant)
  decoders/perceiver.py:7-30 + utils/monkey_patch/blip2_qknorm_monkey_patch.py:37-152   Q-Former with qk LayerNorm
so a reference checkpoint's ``visual_tokenizer.*`` keys load unchanged (HF naming for the CLIP encoder layers and
the BLIP-2 Q-Former).  Arithmetic on the hot spots runs in this repo's kernels: all attention (CLIP patch self-
attention T = 257, 16 x 64; Q-Former self / cross attention 12 x 64) through ``ops.attention`` (wgmma in bf16/f16),
every MSDeformAttn through the sm_90a sampler (D = 32, P = 4, L in {3, 1}), LayerNorms through ``ops.layernorm``;
dense linears / convolutions are library calls (cuBLAS / cuDNN).  The CLIP-encoder and Q-Former arithmetic of the
reference lives in transformers 4.31 / xformers (not under /root/reference): parity for those blocks is checked
against transformers 5.x stand-ins only ("parity unpinned", DESIGN.md section 2).
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import autograd_ops
from . import msda as _msda
from ._cache import WeightCache
from .functions import MSDeformAttnFunction
from .msda import records
from .sd_mmfs import resize_abs_pos, sincos_pos_embed_2d


# ------------------------------------------------------------------------------------------------------
# CLIP ViT encoder (HF naming)
# ------------------------------------------------------------------------------------------------------
class CLIPVisionConfigLite(SimpleNamespace):
    """Fields of HF CLIPVisionConfig used here; defaults = openai/clip-vit-large-patch14."""

    def __init__(self, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                 image_size=224, patch_size=14, layer_norm_eps=1e-5, num_channels=3):
        super().__init__(hidden_size=hidden_size, intermediate_size=intermediate_size,
                         num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                         image_size=image_size, patch_size=patch_size, layer_norm_eps=layer_norm_eps,
                         num_channels=num_channels)


class CLIPVisionEmbeddings(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.embed_dim, self.image_size, self.patch_size = config.hidden_size, config.image_size, config.patch_size
        self.class_embedding = nn.Parameter(torch.randn(self.embed_dim))
        self.patch_embedding = nn.Conv2d(config.num_channels, self.embed_dim, kernel_size=self.patch_size,
                                         stride=self.patch_size, bias=False)
        self.num_patches = (self.image_size // self.patch_size) ** 2
        self.num_positions = self.num_patches + 1
        self.position_embedding = nn.Embedding(self.num_positions, self.embed_dim)
        # persistent like the reference's embeddings (clip_vit_hf.py:85): the key is part of its checkpoints
        self.register_buffer("position_ids", torch.arange(self.num_positions).expand((1, -1)))

    def forward(self, pixel_values):
        B = pixel_values.shape[0]
        patch = self.patch_embedding(pixel_values)                                  # (B, C, Hp, Wp)
        Hp, Wp = patch.shape[2], patch.shape[3]
        patch = patch.flatten(2).transpose(1, 2)
        emb = torch.cat([self.class_embedding.to(patch.dtype).expand(B, 1, -1), patch], dim=1)
        return emb + self.position_embedding.weight[: emb.shape[1]].to(emb.dtype), Hp, Wp   # clip_vit_hf.py:87-96


class CLIPAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.embed_dim, self.num_heads = config.hidden_size, config.num_attention_heads
        self.head_dim = self.embed_dim // self.num_heads
        self.k_proj = nn.Linear(self.embed_dim, self.embed_dim)
        self.v_proj = nn.Linear(self.embed_dim, self.embed_dim)
        self.q_proj = nn.Linear(self.embed_dim, self.embed_dim)
        self.out_proj = nn.Linear(self.embed_dim, self.embed_dim)
        self._qkv = WeightCache()

    def _fused(self):
        ps = (self.q_proj.weight, self.k_proj.weight, self.v_proj.weight, self.q_proj.bias, self.k_proj.bias, self.v_proj.bias)
        return self._qkv.get(ps, lambda: (torch.cat(ps[:3], 0).contiguous(), torch.cat(ps[3:], 0).contiguous()))

    def forward(self, x):
        """softmax(q k^T / sqrt(d)) v, no mask (CLIPXAttention.forward, xattn.py:47-141).  When autograd records the call
        (the gradient of a trainable ViT-Adapter crosses the frozen CLIP layers): forward with the row log-sum-exp and
        the general attention backward into one (B, T, 3, H, hd) gradient, so the fused projection's backward is one
        GEMM.  The q / k / v weights are read through a cache built without grad, so they must be frozen there."""
        if records(self.q_proj, self.k_proj, self.v_proj):
            raise RuntimeError("CLIPAttention: the CLIP q / k / v projections have no weight gradient here (the "
                               "reference freezes the CLIP ViT); freeze them, e.g. with "
                               "VisualTokenizer.freeze_like_reference(), or run under torch.no_grad()")
        B, T, _ = x.shape
        w, b = self._fused()
        qkv = F.linear(x, w, b).view(B, T, 3, self.num_heads, self.head_dim)
        return self.out_proj(autograd_ops.attention(qkv, causal=False))


class CLIPMLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.fc1 = nn.Linear(config.hidden_size, config.intermediate_size)
        self.fc2 = nn.Linear(config.intermediate_size, config.hidden_size)

    def forward(self, x):
        return self.fc2(autograd_ops.quick_gelu(self.fc1(x)))


class CLIPEncoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self_attn = CLIPAttention(config)
        self.layer_norm1 = nn.LayerNorm(config.hidden_size, eps=config.layer_norm_eps)
        self.mlp = CLIPMLP(config)
        self.layer_norm2 = nn.LayerNorm(config.hidden_size, eps=config.layer_norm_eps)

    def forward(self, x):
        n1, n2 = self.layer_norm1, self.layer_norm2
        x = x + self.self_attn(autograd_ops.layernorm(x, n1.weight, n1.bias, n1.eps))
        return x + self.mlp(autograd_ops.layernorm(x, n2.weight, n2.bias, n2.eps))


class CLIPEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.layers = nn.ModuleList([CLIPEncoderLayer(config) for _ in range(config.num_hidden_layers)])


# ------------------------------------------------------------------------------------------------------
# ViT-Adapter
# ------------------------------------------------------------------------------------------------------
class MSDeformAttn(nn.Module):
    """Classic multi-scale deformable attention (vit_adapter/ops/modules/ms_deform_attn.py:27-131)."""

    def __init__(self, d_model=256, n_levels=4, n_heads=8, n_points=4, ratio=1.0):
        super().__init__()
        if d_model % n_heads != 0:
            raise ValueError("d_model must be divisible by n_heads")
        self.im2col_step = 1
        self.d_model, self.n_levels, self.n_heads, self.n_points, self.ratio = d_model, n_levels, n_heads, n_points, ratio
        self.sampling_offsets = nn.Linear(d_model, n_heads * n_levels * n_points * 2)
        self.attention_weights = nn.Linear(d_model, n_heads * n_levels * n_points)
        self.value_proj = nn.Linear(d_model, int(d_model * ratio))
        self.output_proj = nn.Linear(int(d_model * ratio), d_model)
        self._reset_parameters()

    def _reset_parameters(self):
        with torch.no_grad():
            self.sampling_offsets.weight.zero_()
            thetas = torch.arange(self.n_heads, dtype=torch.float32) * (2.0 * math.pi / self.n_heads)
            grid = torch.stack([thetas.cos(), thetas.sin()], -1)
            grid = (grid / grid.abs().max(-1, keepdim=True)[0]).view(self.n_heads, 1, 1, 2).repeat(1, self.n_levels, self.n_points, 1)
            for i in range(self.n_points):
                grid[:, :, i, :] *= i + 1
            self.sampling_offsets.bias.copy_(grid.view(-1))
            self.attention_weights.weight.zero_()
            self.attention_weights.bias.zero_()
            nn.init.xavier_uniform_(self.value_proj.weight)
            self.value_proj.bias.zero_()
            nn.init.xavier_uniform_(self.output_proj.weight)
            self.output_proj.bias.zero_()

    def forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask=None):
        N, Len_q, _ = query.shape
        _, Len_in, _ = input_flatten.shape
        value = self.value_proj(input_flatten)
        if input_padding_mask is not None:
            value = value.masked_fill(input_padding_mask[..., None], float(0))
        value = value.view(N, Len_in, self.n_heads, -1).contiguous()
        off = self.sampling_offsets(query).view(N, Len_q, self.n_heads, self.n_levels, self.n_points, 2)
        aw = self.attention_weights(query).view(N, Len_q, self.n_heads, self.n_levels * self.n_points)
        aw = F.softmax(aw, -1).view(N, Len_q, self.n_heads, self.n_levels, self.n_points)
        if reference_points.shape[-1] != 2:
            raise NotImplementedError("box reference points are not used on this path")
        normalizer = torch.stack([input_spatial_shapes[..., 1], input_spatial_shapes[..., 0]], -1)
        loc = reference_points[:, :, None, :, None, :] + off / normalizer[None, None, None, :, None, :]
        if records(query, input_flatten, self):             # deterministic backward to value, loc and attention weights
            out = MSDeformAttnFunction.apply(value, input_spatial_shapes.contiguous(), input_level_start_index.contiguous(),
                                             loc.to(value.dtype), aw.to(value.dtype), self.im2col_step)
            return self.output_proj(out)
        out = _msda.ms_deform_attn_forward(value, input_spatial_shapes.contiguous(), input_level_start_index.contiguous(),
                                           loc.to(value.dtype).contiguous(), aw.to(value.dtype).contiguous(), self.im2col_step)
        return self.output_proj(out)


class ChannelsFirstLayerNorm(nn.Module):
    """adapter_modules.LayerNorm (channels_first, :236-264): statistics over the channel dim of (B, C, H, W) in fp32."""

    def __init__(self, normalized_shape, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.bias = nn.Parameter(torch.zeros(normalized_shape))
        self.eps = eps

    def forward(self, x):
        return autograd_ops.layernorm(x.permute(0, 2, 3, 1), self.weight, self.bias, self.eps).permute(0, 3, 1, 2)


class SpatialPriorModule(nn.Module):
    def __init__(self, inplanes=64, embed_dim=384, with_cp=False):
        super().__init__()

        def block(cin, cout, stride):
            return [nn.Conv2d(cin, cout, kernel_size=3, stride=stride, padding=1, bias=False), ChannelsFirstLayerNorm(cout),
                    nn.ReLU(inplace=True)]

        self.stem = nn.Sequential(*block(3, inplanes, 2), *block(inplanes, inplanes, 1), *block(inplanes, inplanes, 1),
                                  nn.MaxPool2d(kernel_size=3, stride=2, padding=1))
        self.conv2 = nn.Sequential(*block(inplanes, 2 * inplanes, 2))
        self.conv3 = nn.Sequential(*block(2 * inplanes, 4 * inplanes, 2))
        self.conv4 = nn.Sequential(*block(4 * inplanes, 4 * inplanes, 2))
        self.fc1 = nn.Conv2d(inplanes, embed_dim, kernel_size=1)
        self.fc2 = nn.Conv2d(2 * inplanes, embed_dim, kernel_size=1)
        self.fc3 = nn.Conv2d(4 * inplanes, embed_dim, kernel_size=1)
        self.fc4 = nn.Conv2d(4 * inplanes, embed_dim, kernel_size=1)

    def forward(self, x):
        c1 = self.stem(x)
        c2 = self.conv2(c1)
        c3 = self.conv3(c2)
        c4 = self.conv4(c3)
        c1, c2, c3, c4 = self.fc1(c1), self.fc2(c2), self.fc3(c3), self.fc4(c4)
        bs, dim = c1.shape[:2]
        return c1, c2.view(bs, dim, -1).transpose(1, 2), c3.view(bs, dim, -1).transpose(1, 2), c4.view(bs, dim, -1).transpose(1, 2)


class DWConv(nn.Module):
    def __init__(self, dim=768):
        super().__init__()
        self.dwconv = nn.Conv2d(dim, dim, 3, 1, 1, bias=True, groups=dim)

    def forward(self, x, H, W):
        B, N, C = x.shape
        n = N // 21                                                                  # 16n | 4n | n tokens of the 3 scales
        outs = []
        for sl, (h, w) in ((slice(0, 16 * n), (H * 2, W * 2)), (slice(16 * n, 20 * n), (H, W)), (slice(20 * n, N), (H // 2, W // 2))):
            t = x[:, sl, :].transpose(1, 2).reshape(B, C, h, w)
            outs.append(self.dwconv(t).flatten(2).transpose(1, 2))
        return torch.cat(outs, dim=1)


class ConvFFN(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, drop=0.0):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features or in_features)
        self.dwconv = DWConv(hidden_features or in_features)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden_features or in_features, out_features or in_features)

    def forward(self, x, H, W):
        return self.fc2(self.act(self.dwconv(self.fc1(x), H, W)))


class Extractor(nn.Module):
    def __init__(self, dim, num_heads=6, n_points=4, n_levels=1, deform_ratio=1.0, with_cffn=True, cffn_ratio=0.25, **_):
        super().__init__()
        self.query_norm = nn.LayerNorm(dim, eps=1e-6)
        self.feat_norm = nn.LayerNorm(dim, eps=1e-6)
        self.attn = MSDeformAttn(d_model=dim, n_levels=n_levels, n_heads=num_heads, n_points=n_points, ratio=deform_ratio)
        self.with_cffn = with_cffn
        if with_cffn:
            self.ffn = ConvFFN(in_features=dim, hidden_features=int(dim * cffn_ratio))
            self.ffn_norm = nn.LayerNorm(dim, eps=1e-6)

    def forward(self, query, reference_points, feat, spatial_shapes, level_start_index, H, W):
        qn, fn = self.query_norm, self.feat_norm
        query = query + self.attn(autograd_ops.layernorm(query, qn.weight, qn.bias, qn.eps), reference_points,
                                  autograd_ops.layernorm(feat, fn.weight, fn.bias, fn.eps), spatial_shapes,
                                  level_start_index, None)
        if self.with_cffn:
            n = self.ffn_norm
            query = query + self.ffn(autograd_ops.layernorm(query, n.weight, n.bias, n.eps), H, W)
        return query


class Injector(nn.Module):
    def __init__(self, dim, num_heads=6, n_points=4, n_levels=1, deform_ratio=1.0, init_values=0.0, **_):
        super().__init__()
        self.query_norm = nn.LayerNorm(dim, eps=1e-6)
        self.feat_norm = nn.LayerNorm(dim, eps=1e-6)
        self.attn = MSDeformAttn(d_model=dim, n_levels=n_levels, n_heads=num_heads, n_points=n_points, ratio=deform_ratio)
        self.gamma = nn.Parameter(init_values * torch.ones(dim), requires_grad=True)

    def forward(self, query, reference_points, feat, spatial_shapes, level_start_index):
        qn, fn = self.query_norm, self.feat_norm
        attn = self.attn(autograd_ops.layernorm(query, qn.weight, qn.bias, qn.eps), reference_points,
                         autograd_ops.layernorm(feat, fn.weight, fn.bias, fn.eps), spatial_shapes, level_start_index,
                         None)
        return query + self.gamma * attn


class InteractionBlockWithCls(nn.Module):
    def __init__(self, dim, num_heads=6, n_points=4, with_cffn=True, cffn_ratio=0.25, init_values=0.0, deform_ratio=1.0,
                 extra_extractor=False, **_):
        super().__init__()
        self.injector = Injector(dim=dim, n_levels=3, num_heads=num_heads, init_values=init_values, n_points=n_points,
                                 deform_ratio=deform_ratio)
        self.extractor = Extractor(dim=dim, n_levels=1, num_heads=num_heads, n_points=n_points, deform_ratio=deform_ratio,
                                   with_cffn=with_cffn, cffn_ratio=cffn_ratio)
        self.extra_extractors = nn.Sequential(*[
            Extractor(dim=dim, num_heads=num_heads, n_points=n_points, with_cffn=with_cffn, cffn_ratio=cffn_ratio,
                      deform_ratio=deform_ratio) for _ in range(2)]) if extra_extractor else None

    def forward(self, x, c, cls, blocks, deform_inputs1, deform_inputs2, H, W):
        x = self.injector(x, deform_inputs1[0], c, deform_inputs1[1], deform_inputs1[2])
        x = torch.cat((cls, x), dim=1)
        for blk in blocks:
            x = blk(x)
        cls, x = x[:, :1], x[:, 1:]
        c = self.extractor(c, deform_inputs2[0], x, deform_inputs2[1], deform_inputs2[2], H, W)
        if self.extra_extractors is not None:
            for ext in self.extra_extractors:
                c = ext(c, deform_inputs2[0], x, deform_inputs2[1], deform_inputs2[2], H, W)
        return x, c, cls


def _grid_points(shapes, device):
    pts = []
    for (h, w) in shapes:                                                           # adapter_modules.py:15-27
        ys = (torch.arange(h, device=device, dtype=torch.float32) + 0.5) / h
        xs = (torch.arange(w, device=device, dtype=torch.float32) + 0.5) / w
        gy, gx = torch.meshgrid(ys, xs, indexing="ij")
        pts.append(torch.stack((gx.reshape(-1), gy.reshape(-1)), -1))
    return torch.cat(pts, 0)[None, :, None, :]


def adapter_deform_inputs(h, w, device):
    """adapter_modules.deform_inputs (:30-49) for an (h, w) resized image."""
    def pack(shapes):
        ss = torch.tensor(shapes, dtype=torch.long, device=device)
        return ss, torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
    s3 = [(h // 8, w // 8), (h // 16, w // 16), (h // 32, w // 32)]
    ss1, st1 = pack(s3)
    ss2, st2 = pack([(h // 16, w // 16)])
    return [_grid_points([(h // 16, w // 16)], device), ss1, st1], [_grid_points(s3, device), ss2, st2]


class CLIPVisionTransformerAdapter(nn.Module):
    def __init__(self, config, conv_inplane=64, n_points=4):
        super().__init__()
        self.config = config
        dim = config.hidden_size
        if config.num_hidden_layers % 4 != 0:
            raise NotImplementedError("the adapter splits the encoder into 4 equal stages")
        per = config.num_hidden_layers // 4
        self.interaction_indexes = [[i * per, (i + 1) * per - 1] for i in range(4)]   # [[0,5],[6,11],[12,17],[18,23]] for ViT-L
        self.embeddings = CLIPVisionEmbeddings(config)
        self.pre_layrnorm = nn.LayerNorm(dim, eps=config.layer_norm_eps)
        self.encoder = CLIPEncoder(config)
        self.adapter_level_embed = nn.Parameter(torch.zeros(3, dim))
        self.adapter_spm = SpatialPriorModule(inplanes=conv_inplane, embed_dim=dim)
        self.adapter_interactions = nn.Sequential(*[
            InteractionBlockWithCls(dim=dim, num_heads=config.num_attention_heads, n_points=n_points, init_values=0.0,
                                    with_cffn=True, cffn_ratio=0.25, deform_ratio=0.5, extra_extractor=(i == 3))
            for i in range(4)])
        self.adapter_up = nn.ConvTranspose2d(dim, dim, 2, 2)
        self._geom = {}

    def forward(self, pixel_values):
        cfg = self.config
        hidden, H, W = self.embeddings(pixel_values)
        bs, n, dim = hidden.shape
        pre = self.pre_layrnorm
        hidden = autograd_ops.layernorm(hidden, pre.weight, pre.bias, pre.eps)
        new_size = cfg.image_size // cfg.patch_size * 16                              # vit_adapter_hf.py:113-114
        resized = F.interpolate(pixel_values, size=(new_size, new_size), mode="bilinear", align_corners=False)
        gkey = (new_size, pixel_values.device)
        if gkey not in self._geom:
            self._geom[gkey] = adapter_deform_inputs(new_size, new_size, pixel_values.device)
        d1, d2 = self._geom[gkey]
        c1, c2, c3, c4 = self.adapter_spm(resized)
        c2, c3, c4 = c2 + self.adapter_level_embed[0], c3 + self.adapter_level_embed[1], c4 + self.adapter_level_embed[2]
        c = torch.cat([c2, c3, c4], dim=1)
        x, cls = hidden[:, 1:, :], hidden[:, 0:1, :]
        outs = []
        for i, layer in enumerate(self.adapter_interactions):
            lo, hi = self.interaction_indexes[i]
            x, c, cls = layer(x, c, cls, self.encoder.layers[lo:hi + 1], d1, d2, H, W)
            outs.append(x.transpose(1, 2).reshape(bs, dim, H, W))
        n2, n3 = c2.size(1), c3.size(1)
        c2 = c[:, :n2].transpose(1, 2).reshape(bs, dim, H * 2, W * 2)
        c3 = c[:, n2:n2 + n3].transpose(1, 2).reshape(bs, dim, H, W)
        c4 = c[:, n2 + n3:].transpose(1, 2).reshape(bs, dim, H // 2, W // 2)
        c1 = self.adapter_up(c2) + c1
        x1, x2, x3, x4 = outs
        last_hidden = torch.cat([cls, x4.flatten(2).transpose(1, 2)], dim=1)
        x1 = autograd_ops.resize_bilinear(x1, 4)
        x2 = autograd_ops.resize_bilinear(x2, 2)
        x4 = autograd_ops.resize_bilinear(x4, 0.5)
        return SimpleNamespace(last_hidden_state=last_hidden, pooler_output=cls,
                               hidden_states=[c1 + x1, c2 + x2, c3 + x3, c4 + x4])


class CLIPVisionAdapterModel(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.vision_model = CLIPVisionTransformerAdapter(config)

    def forward(self, pixel_values):
        return self.vision_model(pixel_values)


# ------------------------------------------------------------------------------------------------------
# Q-Former (BLIP-2) with qk LayerNorm
# ------------------------------------------------------------------------------------------------------
class QFormerAttention(nn.Module):
    """Blip2QFormerMultiHeadAttention + qk LayerNorm (blip2_qknorm_monkey_patch.py:37-152), no masks / dropout."""

    def __init__(self, hidden, heads, kv_dim, eps, qk_norm):
        super().__init__()
        self.num_attention_heads, self.attention_head_size = heads, hidden // heads
        self.query = nn.Linear(hidden, hidden)
        self.key = nn.Linear(kv_dim, hidden)
        self.value = nn.Linear(kv_dim, hidden)
        self.q_norm = nn.LayerNorm(self.attention_head_size, eps=eps) if qk_norm else nn.Identity()
        self.k_norm = nn.LayerNorm(self.attention_head_size, eps=eps) if qk_norm else nn.Identity()

    def forward(self, hidden_states, encoder_hidden_states=None, encoder_attention_mask=None):
        """``encoder_attention_mask`` (B, T_kv) 0/1: key padding of the cross-attention (HF adds (1-mask) * finfo.min)."""
        kv = hidden_states if encoder_hidden_states is None else encoder_hidden_states
        B, Tq, _ = hidden_states.shape
        H, hd = self.num_attention_heads, self.attention_head_size
        q = self.query(hidden_states).view(B, Tq, H, hd)
        k = self.key(kv).view(B, kv.shape[1], H, hd)
        v = self.value(kv).view(B, kv.shape[1], H, hd)
        if isinstance(self.q_norm, nn.LayerNorm):
            qn, kn = self.q_norm, self.k_norm
            q = autograd_ops.layernorm(q, qn.weight, qn.bias, qn.eps)
            k = autograd_ops.layernorm(k, kn.weight, kn.bias, kn.eps)
        km = None if (encoder_attention_mask is None or encoder_hidden_states is None) else encoder_attention_mask.to(torch.uint8).contiguous()
        return autograd_ops.attention_general(q, k, v, key_mask=km)      # scores / sqrt(hd), softmax, @ v


class _SelfOutput(nn.Module):
    def __init__(self, hidden, eps):
        super().__init__()
        self.dense = nn.Linear(hidden, hidden)
        self.LayerNorm = nn.LayerNorm(hidden, eps=eps)

    def forward(self, ctx, residual):
        n = self.LayerNorm
        return autograd_ops.layernorm(self.dense(ctx) + residual, n.weight, n.bias, n.eps)


class _AttnBlock(nn.Module):
    def __init__(self, hidden, heads, kv_dim, eps, qk_norm):
        super().__init__()
        self.attention = QFormerAttention(hidden, heads, kv_dim, eps, qk_norm)
        self.output = _SelfOutput(hidden, eps)

    def forward(self, x, enc=None, enc_mask=None):
        return self.output(self.attention(x, enc, enc_mask), x)


class _Intermediate(nn.Module):
    def __init__(self, hidden, inter):
        super().__init__()
        self.dense = nn.Linear(hidden, inter)

    def forward(self, x):
        return F.gelu(self.dense(x))


class _Output(nn.Module):
    def __init__(self, hidden, inter, eps):
        super().__init__()
        self.dense = nn.Linear(inter, hidden)
        self.LayerNorm = nn.LayerNorm(hidden, eps=eps)

    def forward(self, x, residual):
        n = self.LayerNorm
        return autograd_ops.layernorm(self.dense(x) + residual, n.weight, n.bias, n.eps)


class QFormerLayer(nn.Module):
    def __init__(self, cfg, idx):
        super().__init__()
        self.attention = _AttnBlock(cfg.hidden_size, cfg.num_attention_heads, cfg.hidden_size, cfg.layer_norm_eps, cfg.qk_normalization)
        self.has_cross_attention = idx % cfg.cross_attention_frequency == 0
        if self.has_cross_attention:
            self.crossattention = _AttnBlock(cfg.hidden_size, cfg.num_attention_heads, cfg.encoder_hidden_size,
                                             cfg.layer_norm_eps, cfg.qk_normalization)
        self.intermediate_query = _Intermediate(cfg.hidden_size, cfg.intermediate_size)
        self.output_query = _Output(cfg.hidden_size, cfg.intermediate_size, cfg.layer_norm_eps)

    def forward(self, x, enc, enc_mask=None):
        x = self.attention(x)
        if self.has_cross_attention:
            x = self.crossattention(x, enc, enc_mask)
        return self.output_query(self.intermediate_query(x), x)


class _QFormerEncoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.layer = nn.ModuleList([QFormerLayer(cfg, i) for i in range(cfg.num_hidden_layers)])


class Blip2QFormerModel(nn.Module):
    """Query-only path of HF Blip2QFormerModel: layernorm(queries) -> layers -> sequence output."""

    def __init__(self, cfg):
        super().__init__()
        self.config = cfg
        self.layernorm = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)
        self.encoder = _QFormerEncoder(cfg)

    def forward(self, query_embeds, encoder_hidden_states, encoder_attention_mask=None):
        n = self.layernorm
        x = autograd_ops.layernorm(query_embeds, n.weight, n.bias, n.eps)
        for layer in self.encoder.layer:
            x = layer(x, encoder_hidden_states, encoder_attention_mask)
        return x


class PerceiverResampler(nn.Module):
    def __init__(self, num_queries=32, hidden_size=768, qk_normalization=False, encoder_hidden_size=1024,
                 cross_attention_frequency=2, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                 layer_norm_eps=1e-12, **_):
        super().__init__()
        cfg = SimpleNamespace(hidden_size=hidden_size, encoder_hidden_size=encoder_hidden_size,
                              cross_attention_frequency=cross_attention_frequency, num_hidden_layers=num_hidden_layers,
                              num_attention_heads=num_attention_heads, intermediate_size=intermediate_size,
                              layer_norm_eps=layer_norm_eps, qk_normalization=qk_normalization)
        self.blip2qformer = Blip2QFormerModel(cfg)
        self.queries = nn.Parameter(torch.zeros(1, num_queries, hidden_size).normal_(0, 0.02))

    def forward(self, encoder_hidden_states, query_embeds=None, encoder_attention_mask=None, **_):
        q = self.queries if query_embeds is None else query_embeds
        q = q.to(encoder_hidden_states.dtype).expand(encoder_hidden_states.shape[0], -1, -1)
        return (self.blip2qformer(q, encoder_hidden_states, encoder_attention_mask),)


# ------------------------------------------------------------------------------------------------------
# VisualTokenizer
# ------------------------------------------------------------------------------------------------------
CLIP_MEAN, CLIP_STD = [0.48145466, 0.4578275, 0.40821073], [0.26862954, 0.26130258, 0.27577711]


class VisualTokenizer(nn.Module):
    def __init__(self, encoder_model_path=None, perceiver_config=None, llm_hidden_size=5120, clip_normalize=True,
                 grid_size=16, clip_config=None):
        """Reference constructor arguments (visual_tokenizer.py:12-19).  ``encoder_model_path`` is only consulted for
        its ``config.json`` (vision_config fields); weights arrive through ``load_state_dict`` like in the reference's
        ``load_model_weights`` (utils/misc.py:13-63).  ``clip_config`` (extension) overrides it."""
        super().__init__()
        if clip_config is None:
            clip_config = CLIPVisionConfigLite()
            cfg_file = None if encoder_model_path is None else __import__("os").path.join(str(encoder_model_path), "config.json")
            if cfg_file and __import__("os").path.exists(cfg_file):
                import json
                raw = json.load(open(cfg_file))
                raw = raw.get("vision_config", raw)
                for k in ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "image_size",
                          "patch_size", "layer_norm_eps"):
                    if k in raw:
                        setattr(clip_config, k, raw[k])
        if perceiver_config is None:
            perceiver_config = dict(num_queries=64, hidden_size=768, encoder_hidden_size=1024, cross_attention_frequency=2,
                                    num_hidden_layers=12, num_attention_heads=12, qk_normalization=True)
        perceiver_config = dict(perceiver_config) if not isinstance(perceiver_config, dict) else dict(perceiver_config)
        self.clip_normalize = clip_normalize
        self.encoder = CLIPVisionAdapterModel(clip_config)
        enc = perceiver_config["encoder_hidden_size"]
        self.pos_proj = nn.Linear(enc, enc)
        self.pos_ln = nn.LayerNorm(enc, eps=1e-6)
        pe = torch.cat([torch.zeros(1, enc), sincos_pos_embed_2d(enc, grid_size)], 0)       # cls_token=True (:27-31)
        self.pos_embed = nn.Parameter(pe, requires_grad=False)
        self._abs_pos_cache = WeightCache()
        self.perceiver_resampler = PerceiverResampler(**perceiver_config)
        self.length = perceiver_config["num_queries"]
        self.post_ln = nn.LayerNorm(enc, eps=1e-6)
        self.proj = nn.Linear(perceiver_config["hidden_size"], llm_hidden_size)
        nn.init.normal_(self.proj.weight, std=1.0e-3)
        nn.init.zeros_(self.proj.bias)
        if clip_normalize:
            self.register_buffer("clip_mean", torch.tensor(CLIP_MEAN).view(1, 3, 1, 1))
            self.register_buffer("clip_std", torch.tensor(CLIP_STD).view(1, 3, 1, 1))

    def freeze_like_reference(self):
        """The trainable set of the reference's tokenizer (vit_adapter_hf.py:246-252 with freeze=False, freeze_vit=True;
        visual_tokenizer.py:27-31): in the encoder only the ViT-Adapter (parameters of ``encoder.vision_model`` whose
        name starts with ``adapter``: the spatial prior module, injectors, extractors, ``adapter_level_embed``,
        ``adapter_up``), the whole head (``pos_proj``, ``pos_ln``, the Q-Former, ``post_ln``, ``proj``), and not the
        fixed ``pos_embed`` table.  The CLIP ViT stays frozen; its layers still pass the adapter's gradient on.
        Returns ``self``.  ``MMInterleaved.freeze_like_reference()`` leaves the tokenizer alone: call both to train
        like the reference, ``model.freeze_like_reference(); model.visual_tokenizer.freeze_like_reference()``."""
        for name, p in self.encoder.vision_model.named_parameters():
            p.requires_grad_(name.startswith("adapter"))
        for name, p in self.named_parameters():
            if not name.startswith("encoder."):
                p.requires_grad_(name != "pos_embed")
        return self

    def abs_pos(self, n):
        """``pos_embed`` without its cls row, resized to ``n`` positions.  Cached per length on the parameter itself
        (the reference re-interpolates on every forward); not while the table is being trained."""
        if torch.is_grad_enabled() and self.pos_embed.requires_grad:
            return resize_abs_pos(self.pos_embed[1:], n)
        return self._abs_pos_cache.get(self.pos_embed, lambda: resize_abs_pos(self.pos_embed[1:], n), key=n)

    def forward(self, image):
        if self.clip_normalize:
            image = (image - self.clip_mean.to(image.dtype)) / self.clip_std.to(image.dtype)
        out = self.encoder(image)
        image_embed = out.last_hidden_state
        feats = []
        for f in out.hidden_states:                                                       # :74-82
            pe = self.abs_pos(f.size(2) * f.size(3))
            feats.append(f + pe.to(f.dtype).view(f.size(2), f.size(3), -1).permute(2, 0, 1))
        n = image_embed.size(1)
        pe = torch.cat([self.pos_embed[:1], self.abs_pos(n - 1)], 0).to(image_embed.dtype)
        pn, qn = self.pos_ln, self.post_ln
        q_in = autograd_ops.layernorm(self.pos_proj(image_embed), pn.weight, pn.bias, pn.eps) + pe      # :85-87
        image_embed = image_embed + pe
        q_in = autograd_ops.layernorm(q_in, qn.weight, qn.bias, qn.eps)
        vis = self.perceiver_resampler(encoder_hidden_states=q_in)[0]
        return dict(vis_embed=self.proj(vis), image_embeds=image_embed[:, 1:, :], multiscale_features=feats)
