"""``MMFS`` -- Multi-Image Multi-Scale Feature Synchronizer, H100-native.

Drop-in for the reference module ``mm_interleaved.models.utils.ops.modules.mmfs.MMFS``
(ops/modules/mmfs.py:25-276): same constructor arguments, same parameter / state-dict names
(``sampling_offsets``, ``ignore_token``, ``dynamic_offset_mask``, ``attention_weights``,
``value_proj``, ``output_proj``, ``query_relpos``; mmfs.py:85-96), same ``forward`` signature
(mmfs.py:120-129).  It is NOT a translation of the reference forward:

* ``dynamic_offset_mask`` runs once per token instead of once per (token, image) -- the reference
  repeats the query n_images times before the 5120x5120 linear (mmfs.py:174-175);
* the per-image conditioning ``Linear(q1 + relpos_embed[r])`` (mmfs.py:178-191) is factored by
  linearity into ``Linear(q1)`` (one GEMM producing offsets and logits for all heads) plus a
  ``(max_num_image_per_seq, C)`` table ``W @ relpos_embed`` looked up inside the sampler kernel;
* mask add, null-slot softmax, location arithmetic and the deformable gather are one sm_90a
  kernel (csrc/mmfs_sampler_sm100.cu); the (N,Lq,M,L,P,2) / (N,Lq,M,L,P) tensors never exist;
* ``value_proj(input_flatten)`` is cached while the same feature tensor is passed again (decode
  steps, denoise steps) -- the reference recomputes it every call (mmfs.py:165).

Dense projections are cuBLAS GEMMs through ``torch.nn.functional.linear``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn

from . import msda as _msda
from . import sampler as _sampler
from ._cache import SourceCache

_FAST_HEAD_DIMS = (32, 64, 128)


_RELPOS_CACHE = {}


def relative_image_index(attention_mask: torch.Tensor, len_q: int) -> torch.Tensor:
    """uint8 (N, n_img, 1|Lq): newest visible image -> 1, older -> 2.., masked -> 0 (mmfs.py:154-163).
    Every MMFS layer of a forward receives the same mask tensor, so the last result is kept (keyed on the
    tensor's storage + version) instead of being recomputed per layer."""
    key = (attention_mask.data_ptr(), attention_mask._version, tuple(attention_mask.shape), attention_mask.dtype,
           attention_mask.device, len_q)
    hit = _RELPOS_CACHE.get("last")
    if hit is not None and hit[0] == key and hit[1]() is attention_mask:
        return hit[2]
    rel = _relative_image_index(attention_mask, len_q)
    if not torch.is_grad_enabled() or not attention_mask.requires_grad:
        import weakref
        _RELPOS_CACHE["last"] = (key, weakref.ref(attention_mask), rel)
    return rel


def _relative_image_index(attention_mask: torch.Tensor, len_q: int) -> torch.Tensor:
    m = attention_mask.long()
    tot = m.sum(dim=-1, keepdim=True)
    rel = (tot + 1 - m.cumsum(dim=-1)) * m
    if attention_mask.ndim == 2:
        rel = rel.unsqueeze(-1)                                  # (N, n, 1): same for every query
    else:
        if attention_mask.shape[1] != len_q:
            rel = rel[:, -1:, :]                                 # decode step: last mask row
        rel = rel.transpose(1, 2)                                # b q n -> b n q
    return rel.to(torch.uint8).contiguous()


class MMFS(nn.Module):
    def __init__(self, layer_idx=0, d_model=256, d_query=-1, d_value=256, d_out=-1, n_levels=4, n_heads=8,
                 n_points=8, ratio=1.0, offset_init_magnitude=3, spatial_shapes=[16], base_spatial_shape=16,
                 max_num_image_per_seq=50):
        super().__init__()
        if d_model % n_heads != 0:
            raise ValueError("d_model must be divisible by n_heads, but got {} and {}".format(d_model, n_heads))
        if d_query < 0:
            d_query = d_model
        if d_out < 0:
            d_out = d_model
        self.layer_idx = layer_idx
        self.im2col_step = 1
        self.d_model, self.n_levels, self.n_heads, self.n_points = d_model, n_levels, n_heads, n_points
        self.ratio = ratio
        self.offset_init_magnitude = offset_init_magnitude
        self.max_num_image_per_seq = max_num_image_per_seq
        assert len(spatial_shapes) == n_levels
        self._scale_list = [s / base_spatial_shape for s in spatial_shapes]   # to rebuild the buffer after to_empty()
        self.register_buffer("scale_ratios", torch.tensor([s / base_spatial_shape for s in spatial_shapes]),
                             persistent=False)
        d_inner = int(d_model * ratio)
        self.sampling_offsets = nn.Linear(d_query, n_heads * n_points * 2)
        self.ignore_token = nn.Parameter(torch.zeros(1, 1, 1, d_inner), requires_grad=False)
        self.dynamic_offset_mask = nn.Linear(d_query, d_query)
        self.attention_weights = nn.Linear(d_query, n_heads * n_levels * (n_points + 1))
        self.value_proj = nn.Linear(d_value, d_inner)
        self.output_proj = nn.Linear(d_inner, d_out)
        self.query_relpos = nn.Embedding(max_num_image_per_seq, d_query)
        self._reset_parameters()
        self._fused = None        # (versions, W_cat, b_cat, rtable)
        self._value_cache = SourceCache()  # value_proj(input_flatten), identity-checked (see _cache.py)

    def _reset_parameters(self):   # same initialisation scheme as mmfs.py:102-118
        grid = torch.empty(self.n_heads, 1, self.n_points, 2).uniform_(-self.offset_init_magnitude,
                                                                      self.offset_init_magnitude)
        with torch.no_grad():
            self.sampling_offsets.weight.zero_()
            self.sampling_offsets.bias.copy_(grid.view(-1))
            self.attention_weights.bias.zero_()
            nn.init.xavier_uniform_(self.value_proj.weight)
            self.value_proj.bias.zero_()
            nn.init.xavier_uniform_(self.output_proj.weight)
            self.output_proj.bias.zero_()
            self.dynamic_offset_mask.bias.zero_()
            nn.init.trunc_normal_(self.query_relpos.weight, std=0.02)

    # -- cached derived weights -----------------------------------------------------------------------
    def _fused_weights(self):
        ps = (self.sampling_offsets.weight, self.sampling_offsets.bias, self.attention_weights.weight,
              self.attention_weights.bias, self.query_relpos.weight)
        key = tuple((p.data_ptr(), p._version, p.dtype, p.device) for p in ps)
        if self._fused is None or self._fused[0] != key:
            with torch.no_grad():
                w = torch.cat([ps[0], ps[2]], 0).contiguous()
                b = torch.cat([ps[1], ps[3]], 0).contiguous()
                rtable = F.linear(ps[4], w).contiguous()          # W @ relpos_embed[r], no bias
            self._fused = (key, w, b, rtable)
        return self._fused[1:]

    def project_value(self, input_flatten, input_padding_mask=None, cache=True):
        """value_proj(input_flatten) as (N, n_img*hw, M, D), cached per input tensor (mmfs.py:165-172).  ``cache=False``:
        compute only (callers that keep the result themselves, e.g. ``MMFSNet.prepare``)."""
        w, b = self.value_proj.weight, self.value_proj.bias
        extra = (w.data_ptr(), w._version, b.data_ptr(), b._version)
        cacheable = cache and input_padding_mask is None and not torch.is_grad_enabled()
        if cacheable:
            hit = self._value_cache.get(input_flatten, extra)
            if hit is not None:
                return hit
        N, n_img, hw, _ = input_flatten.shape
        value = self.value_proj(input_flatten)
        if input_padding_mask is not None:
            value = value.masked_fill(input_padding_mask[..., None], float(0))
        value = value.reshape(N, n_img * hw, self.n_heads, value.shape[-1] // self.n_heads).contiguous()
        if cacheable:
            self._value_cache.put(input_flatten, value, extra)
        return value

    def forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask=None, attention_mask=None, output_weight=None, output_bias=None, value=None):
        """Reference signature (mmfs.py:120-129).  ``output_weight`` / ``output_bias`` (extension) replace
        ``output_proj`` for callers that fold a following linear map into it (MMFSBlock's 1x1 conv); ``value``
        (extension) supplies value_proj(input_flatten) computed by the caller (``input_flatten`` may then be None)."""
        N, Len_q, _ = query.shape
        assert attention_mask is not None and attention_mask.ndim in (2, 3)
        n_images = attention_mask.shape[-1]
        if input_flatten is not None:
            assert input_flatten.shape[1] == n_images
        if input_spatial_shapes.shape[0] != n_images * self.n_levels:
            raise RuntimeError("input_spatial_shapes must list n_images * n_levels levels")
        if n_images >= self.max_num_image_per_seq:
            # the relative image index of a token reaches n_images and indexes query_relpos / the W e_r table; the
            # reference asserts image_relpos.max() < max_num_image_per_seq (mmfs.py:177) after a device sync
            raise RuntimeError(f"MMFS: {n_images} images per sequence need max_num_image_per_seq > {n_images} "
                               f"(got {self.max_num_image_per_seq})")
        if reference_points.shape[-1] != 2:
            # the box form (mmfs.py:251-258) is not used by any caller on the interleaved forward path
            raise NotImplementedError("MMFS (H100): only 2-D reference points are implemented")
        if not query.is_cuda:
            raise RuntimeError("MMFS (H100) runs on CUDA tensors only (no CPU fallback)")

        if value is None:
            value = self.project_value(input_flatten, input_padding_mask)
        relpos = relative_image_index(attention_mask, Len_q)
        w_cat, b_cat, rtable = self._fused_weights()
        q1 = self.dynamic_offset_mask(query)                       # once per token
        qproj = F.linear(q1, w_cat, b_cat).contiguous()            # offsets | logits for all heads
        ref = reference_points.to(torch.float32)
        if ref.dim() != 4:
            raise RuntimeError("reference_points must be (N|1, Lq, L|1, 2)")
        ref = ref.contiguous()
        shapes = input_spatial_shapes.contiguous()
        starts = input_level_start_index.contiguous()
        scale = self.scale_ratios.to(torch.float32).contiguous()
        ign_key = (self.ignore_token.data_ptr(), self.ignore_token._version)
        if self._ignore_nonzero is None or self._ignore_nonzero[0] != ign_key:   # one host sync per weight load
            self._ignore_nonzero = (ign_key, bool(torch.count_nonzero(self.ignore_token)))
        need_null = self._ignore_nonzero[1]

        D = value.shape[-1]
        if D in _FAST_HEAD_DIMS:
            res = _sampler.mmfs_sampler_forward(value, shapes, starts, qproj, rtable, relpos, ref, scale,
                                                self.n_levels, self.n_points, want_null_mass=need_null)
            sampled, null_mass = res if need_null else (res, None)
        else:   # head sizes without a fused gather: materialise loc / weights, then the generic op
            loc, attn, null_mass = _sampler.mmfs_sampler_locw(shapes, starts, qproj, rtable, relpos, ref, scale,
                                                              self.n_heads, self.n_levels, self.n_points)
            sampled = _msda.ms_deform_attn_forward(value, shapes, starts, loc, attn, self.im2col_step)
        if need_null:   # ignore-token term, mmfs.py:236-241 (a frozen zeros parameter unless a checkpoint sets it)
            ign = self.ignore_token.view(1, 1, self.n_heads, -1).to(sampled.dtype)
            sampled = sampled + (ign * null_mass.unsqueeze(-1).to(sampled.dtype)).reshape(N, Len_q, -1)
        if output_weight is not None:
            return F.linear(sampled, output_weight, output_bias)
        return self.output_proj(sampled)

    _ignore_nonzero = None   # cache of (key, "ignore_token has non-zero entries")

    def _load_from_state_dict(self, *args, **kwargs):
        super()._load_from_state_dict(*args, **kwargs)
        self._fused = None
        self._value_cache.clear()
        self._ignore_nonzero = None
