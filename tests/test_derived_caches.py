"""Values derived from weights (fused matrices, re-laid-out filters, resized position tables, ...) are cached and must be
rebuilt whenever a source changes in any of the ways a model's weights change: an in-place ``load_state_dict``, a
``load_state_dict(assign=True)`` whose new parameters carry the old version numbers, ``p.data = t`` and ``.double()``
(the last two keep the Parameter object and its version).  CPU only: every getter below runs without a device."""
import pytest
import torch
import torch.nn.functional as F

import mm_interleaved_b200 as m
from mm_interleaved_b200 import ops, unet_sd, visual_tokenizer as vt
from mm_interleaved_b200._cache import WeightCache, clear_activation_caches
from mm_interleaved_b200.llama_mmfs import LlamaMLP, LlamaMMFSAttention, LlamaMMFSConfig
from mm_interleaved_b200.mm_interleaved import TextDecoder
from mm_interleaved_b200.mmfs import _relative_image_index, relative_image_index
from mm_interleaved_b200.sd_mmfs import MMFSBlock, pixel_reference_points, resize_abs_pos
from tests.golden.make_golden import TOKENIZER_TINY


def _equal(a, b):
    if torch.is_tensor(a):
        return torch.is_tensor(b) and a.dtype == b.dtype and torch.equal(a, b)
    if isinstance(a, tuple):
        return isinstance(b, tuple) and len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return a == b


def _random_like(t, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(t.shape, generator=g, dtype=t.dtype) if t.is_floating_point() else t.clone()


def _text_head():
    return TextDecoder(hidden_size=16, vocab_size=260, orig_vocab_size=256)


def _text_head_ref(mod):
    w, b = mod.head.weight, mod.head.bias
    tail_w = torch.cat([w[:256], w[256:] + mod.head_new.weight])
    tail_b = torch.cat([b[:256], b[256:] + mod.head_new.bias])
    return F.pad(tail_w, (0, 0, 0, 124)), F.pad(tail_b, (0, 124))


def _clip_attention():
    return vt.CLIPAttention(vt.CLIPVisionConfigLite(hidden_size=32, num_attention_heads=2))


def _clip_ref(mod):
    return (torch.cat([mod.q_proj.weight, mod.k_proj.weight, mod.v_proj.weight]),
            torch.cat([mod.q_proj.bias, mod.k_proj.bias, mod.v_proj.bias]))


def _mmfs_attention():
    cfg = LlamaMMFSConfig(hidden_size=64, intermediate_size=128, num_attention_heads=4, image_embed_dim=64,
                          spatial_shapes=[4, 2])
    return LlamaMMFSAttention(cfg, 0)


def _gated_ref(mod):
    t = mod.gate.float().tanh()
    w, b = mod.attn.output_proj.weight, mod.attn.output_proj.bias
    return (w.float() * t).to(w.dtype), (b.float() * t).to(b.dtype)


def _mmfs():
    return m.MMFS(d_model=32, d_value=24, n_levels=2, n_heads=2, n_points=2, spatial_shapes=[4, 2],
                  max_num_image_per_seq=4)


def _mmfs_ref(mod):
    w = torch.cat([mod.sampling_offsets.weight, mod.attention_weights.weight])
    return w, torch.cat([mod.sampling_offsets.bias, mod.attention_weights.bias]), F.linear(mod.query_relpos.weight, w)


_FEAT = {torch.float32: torch.randn(1, 2, 20, 24)}     # one feature tensor object per dtype


def _feat(dtype):
    return _FEAT.setdefault(dtype, _FEAT[torch.float32].to(dtype))


def _project(mod):
    return mod.project_value(_feat(mod.value_proj.weight.dtype))


def _project_ref(mod):
    return mod.value_proj(_feat(mod.value_proj.weight.dtype)).reshape(1, 40, 2, 16)


def _block():
    return MMFSBlock(attn_dim=64, query_dim=64, feat_dim=64, num_heads=2, grid_size=8, spatial_shapes=[4])


def _geometry(mod):
    return mod._geometry(torch.device("cpu"), torch.float32, 4, 4, 1, [(4, 4)])


def _geometry_ref(mod):
    pos = F.interpolate(mod.pos_embed.float().reshape(1, 8, 8, -1).permute(0, 3, 1, 2), size=(4, 4), mode="bicubic",
                        align_corners=False).permute(0, 2, 3, 1).flatten(0, 2).float()
    return pixel_reference_points(4, 4, "cpu"), torch.tensor([[4, 4]]), torch.tensor([0]), pos


def _out_conv_ref(mod):
    wc = mod.conv.weight.view(64, 64).float()
    wo, bo = mod.mmfs.output_proj.weight, mod.mmfs.output_proj.bias
    return (wc @ wo.float()).to(wo.dtype), (wc @ bo.float() + mod.conv.bias.float()).to(wo.dtype)


def _tokenizer():
    c = TOKENIZER_TINY
    return vt.VisualTokenizer(clip_config=vt.CLIPVisionConfigLite(**c["clip"]), perceiver_config=dict(c["perceiver"]),
                              llm_hidden_size=c["llm_hidden_size"], grid_size=c["grid_size"])


def _abs_pos_ref(mod, n):
    return resize_abs_pos(mod.pos_embed[1:].detach().clone(), n)


GETTERS = {
    "TextDecoder._fused": (_text_head, lambda mod: mod._fused(), _text_head_ref),
    "CLIPAttention._fused": (_clip_attention, lambda mod: mod._fused(), _clip_ref),
    "_CatWeight.get": (lambda: LlamaMLP(16, 24, "silu"), lambda mod: mod._gate_up.get(),
                       lambda mod: torch.cat([mod.gate_proj.weight, mod.up_proj.weight])),
    "LlamaMMFSAttention._gated_output": (_mmfs_attention, lambda mod: mod._gated_output(), _gated_ref),
    "MMFS._fused_weights": (_mmfs, lambda mod: mod._fused_weights(), _mmfs_ref),
    "MMFS.project_value": (_mmfs, _project, _project_ref),
    "MMFSBlock._geometry": (_block, _geometry, _geometry_ref),
    "MMFSBlock._out_conv_fused": (_block, lambda mod: mod._out_conv_fused(), _out_conv_ref),
    "VisualTokenizer.abs_pos": (_tokenizer, lambda mod: mod.abs_pos(4), lambda mod: _abs_pos_ref(mod, 4)),
    "Conv2d.weight_khwc": (lambda: unet_sd.Conv2d(8, 16, 3, padding=1), lambda mod: mod.weight_khwc(),
                           lambda mod: mod.weight.permute(0, 2, 3, 1).contiguous()),
    "Conv2d.weight_up2x": (lambda: unet_sd.Conv2d(8, 16, 3, padding=1), lambda mod: mod.weight_up2x(),
                           lambda mod: ops.fold_up2x_weights(mod.weight)),
}


@pytest.mark.parametrize("name", list(GETTERS))
def test_derived_value_is_rebuilt_whenever_a_source_changes(name):
    make, get, ref = GETTERS[name]
    torch.manual_seed(0)
    mod = make()
    state = [None]

    def check_rebuilt(step):
        new = get(mod)
        assert new is not state[0], step                    # a miss ...
        assert _equal(new, ref(mod)), step                  # ... that equals a from-scratch computation
        assert get(mod) is new, step                        # and is reused afterwards
        state[0] = new

    with torch.no_grad():
        state[0] = get(mod)
        assert get(mod) is state[0]                         # a repeated call is a hit
        assert _equal(state[0], ref(mod))
        mod.load_state_dict({k: _random_like(v, 1) for k, v in mod.state_dict().items()})
        check_rebuilt("in-place load_state_dict")

        sd = {k: _random_like(v, 2) for k, v in mod.state_dict().items()}
        params = dict(mod.named_parameters())
        for k, t in sd.items():                             # the new objects carry the old version numbers
            while k in params and t._version < params[k]._version:
                t.add_(0)
        mod.load_state_dict(sd, assign=True)
        assert all(p._version == params[k]._version for k, p in mod.named_parameters())
        check_rebuilt("load_state_dict(assign=True)")

        for i, (k, p) in enumerate(mod.named_parameters()):
            version = p._version
            p.data = _random_like(p, 3 + i)
            assert p._version == version
        check_rebuilt("p.data = t")

        mod.double()
        check_rebuilt(".double()")


def test_geometry_follows_a_reassigned_position_table():
    """The position table of an MMFSBlock, reloaded with ``assign=True``: the new Parameter has the same version (0)."""
    b = _block()
    old = _geometry(b)[3].clone()
    sd = {k: v.clone() for k, v in b.state_dict().items()}
    sd["pos_embed"] = torch.randn_like(sd["pos_embed"])
    b.load_state_dict(sd, assign=True)
    new = _geometry(b)[3]
    assert not torch.equal(new, old)
    assert torch.equal(new, _geometry_ref(b)[3])


def test_ignore_token_check_follows_reloads():
    mod = _mmfs()
    assert mod._needs_null_slot() is False
    mod.load_state_dict({**mod.state_dict(), "ignore_token": torch.ones(1, 1, 1, 32)})
    assert mod._needs_null_slot() is True
    mod.load_state_dict({**mod.state_dict(), "ignore_token": torch.zeros(1, 1, 1, 32)}, assign=True)
    assert mod._needs_null_slot() is False
    mod.ignore_token.data = torch.full((1, 1, 1, 32), 2.0)
    assert mod._needs_null_slot() is True


def test_resized_position_table_is_cached_per_length_on_the_parameter():
    """``pos_embed[1:]`` is a new view object on every forward: the cache must key on the Parameter, and hold every
    length one forward asks for (one per multi-scale feature level plus the patch count)."""
    tok = _tokenizer()
    with torch.no_grad():
        tables = {n: tok.abs_pos(n) for n in (64, 16, 4, 1)}
        for n, t in tables.items():
            assert tok.abs_pos(n) is t
            assert torch.equal(t, resize_abs_pos(tok.pos_embed[1:], n))
    tok.pos_embed.requires_grad_(True)
    assert tok.abs_pos(64).requires_grad                   # trained table: recomputed with autograd, not cached


def test_relative_image_index_is_shared_until_the_mask_changes():
    mask = torch.tensor([[1, 0, 1, 1]])
    rel = relative_image_index(mask, 5)
    assert relative_image_index(mask, 5) is rel
    assert relative_image_index(mask, 3) is not rel
    mask[0, 1] = 1
    assert torch.equal(relative_image_index(mask, 5), _relative_image_index(mask, 5))


def test_weight_caches_survive_clear_activation_caches():
    """Captured CUDA graphs read weight-derived tensors: dropping them would free memory a graph still reads."""
    mod = _mmfs()
    w = mod._fused_weights()
    clear_activation_caches(mod)
    assert mod._fused_weights() is w
    assert isinstance(mod._fused, WeightCache)
