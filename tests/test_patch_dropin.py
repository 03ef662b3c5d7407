"""The reference's ``replace_*()`` start-up mechanism (inference.py:10-24) pointed at this repository's classes.
``replace_*_b200()`` finds the reference modules by name in ``sys.modules``, so stand-in modules registered under the
reference's module names exercise every rebinding and ``restore_reference()``.  Checkpoint compatibility: the
substituted modules, and the top-level ``MMInterleaved``, have exactly the reference's state-dict layout (names and
shapes), so a checkpoint saved from the reference loads with ``strict=True``; the reference layouts (``LlamaModel`` and
``MMFSNet`` at the tiny test configurations) are stored in tests/golden/reference_checks.npz by
tests/golden/make_golden.py.  CPU-only (construction + state-dict load; compute needs the GPU)."""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_checks.npz")


def _ref_layout(name):
    return {k: tuple(v) for k, v in json.loads(str(np.load(GOLDEN)[f"layout_{name}"])).items()}


def _zeros(layout):
    return {k: torch.zeros(v) for k, v in layout.items()}


def _stub_reference(monkeypatch):
    """Stand-ins for the reference modules patch.py rebinds, registered under the reference's module names: each
    defines the reference's class names, ``sd_mmfs`` / ``ops.modules`` hold second bindings of ``MMFS`` the way
    ``from ..x import MMFS`` creates them, and ``modeling_llama_mmfs.build_layer`` is reference-style glue that looks
    the layer class up in its module at call time."""
    def mod(name, **attrs):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        monkeypatch.setitem(sys.modules, name, m)
        return m

    cls = {n: type(n, (), {}) for n in ("MMFS", "LlamaRMSNorm", "LlamaMLP", "LlamaAttention", "LlamaMMFSAttention",
                                         "LlamaDecoderLayer", "MMFSNet", "MMFSBlock", "VisualTokenizer",
                                         "PerceiverResampler")}
    ns = types.SimpleNamespace(cls=cls, ext=types.ModuleType("MultiScaleDeformableAttention"))   # the compiled op
    mod("mm_interleaved")
    ns.msda_func = mod("mm_interleaved.models.utils.ops.functions.ms_deform_attn_func", MSDA=ns.ext)
    ns.msda_func_vit = mod("mm_interleaved.models.encoders.vit_adapter.ops.functions.ms_deform_attn_func", MSDA=ns.ext)
    ns.mmfs = mod("mm_interleaved.models.utils.ops.modules.mmfs", MMFS=cls["MMFS"])
    ns.ops_modules = mod("mm_interleaved.models.utils.ops.modules", MMFS=cls["MMFS"])
    ns.llama = mod("mm_interleaved.models.decoders.modeling_llama_mmfs",
                   **{n: cls[n] for n in ("LlamaRMSNorm", "LlamaMLP", "LlamaAttention", "LlamaMMFSAttention",
                                          "LlamaDecoderLayer")})
    exec("def build_layer():\n    return LlamaDecoderLayer", vars(ns.llama))
    ns.sd_mmfs = mod("mm_interleaved.models.decoders.sd_mmfs", MMFS=cls["MMFS"], MMFSNet=cls["MMFSNet"],
                     MMFSBlock=cls["MMFSBlock"])
    ns.tokenizer = mod("mm_interleaved.models.encoders.visual_tokenizer", VisualTokenizer=cls["VisualTokenizer"])
    ns.perceiver = mod("mm_interleaved.models.decoders.perceiver", PerceiverResampler=cls["PerceiverResampler"])
    monkeypatch.delitem(sys.modules, "MultiScaleDeformableAttention", raising=False)
    return ns


def test_replace_functions_rebind_the_reference_and_checkpoints_load(monkeypatch):
    """``replace_*_b200()`` rebinds every reference binding of the substituted classes (including second bindings and
    the ``MultiScaleDeformableAttention`` extension module), reference glue then builds this repository's classes,
    ``restore_reference()`` undoes all of it, and reference checkpoints load into the substituted modules with
    ``strict=True``."""
    import mm_interleaved_b200 as b200
    from mm_interleaved_b200 import patch
    from tests.golden.make_golden import LLAMA_TINY, MMFSNET_TINY
    ns = _stub_reference(monkeypatch)
    c = ns.cls
    try:
        b200.replace_mmfs_b200()
        assert ns.mmfs.MMFS is b200.MMFS and ns.sd_mmfs.MMFS is b200.MMFS and ns.ops_modules.MMFS is b200.MMFS
        ext = sys.modules["MultiScaleDeformableAttention"]
        assert ext.ms_deform_attn_forward is b200.ms_deform_attn_forward
        assert ns.msda_func.MSDA is ext and ns.msda_func_vit.MSDA is ext

        b200.replace_llama_b200()
        for name in ("LlamaRMSNorm", "LlamaMLP", "LlamaAttention", "LlamaMMFSAttention", "LlamaDecoderLayer"):
            assert getattr(ns.llama, name) is getattr(b200, name)
        assert ns.llama.build_layer() is b200.LlamaDecoderLayer      # the reference's glue now builds this repo's layer

        b200.replace_visual_b200()
        assert ns.sd_mmfs.MMFSNet is b200.MMFSNet and ns.sd_mmfs.MMFSBlock is b200.MMFSBlock
        assert ns.tokenizer.VisualTokenizer is b200.visual_tokenizer.VisualTokenizer
        assert ns.perceiver.PerceiverResampler is b200.visual_tokenizer.PerceiverResampler

        b200.replace_all_b200()                                           # idempotent
        assert ns.llama.LlamaDecoderLayer is b200.LlamaDecoderLayer and ns.mmfs.MMFS is b200.MMFS
    finally:
        patch.restore_reference()
    assert ns.mmfs.MMFS is c["MMFS"] and ns.sd_mmfs.MMFS is c["MMFS"] and ns.ops_modules.MMFS is c["MMFS"]
    assert ns.llama.LlamaDecoderLayer is c["LlamaDecoderLayer"] and ns.llama.build_layer() is c["LlamaDecoderLayer"]
    assert ns.sd_mmfs.MMFSNet is c["MMFSNet"] and ns.tokenizer.VisualTokenizer is c["VisualTokenizer"]
    assert ns.msda_func.MSDA is ns.ext and ns.msda_func_vit.MSDA is ns.ext
    assert "MultiScaleDeformableAttention" not in sys.modules

    # checkpoints: the substituted modules have exactly the reference's state-dict layout
    ref_llama, ref_net = _ref_layout("llama"), _ref_layout("mmfsnet")
    model = b200.LlamaModel(b200.LlamaMMFSConfig(**LLAMA_TINY))
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == ref_llama
    missing, unexpected = model.load_state_dict(_zeros(ref_llama), strict=True)
    assert not missing and not unexpected
    net = b200.MMFSNet(**MMFSNET_TINY)
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == ref_net
    net.load_state_dict(_zeros(ref_net), strict=True)


def test_b200_top_level_model_keeps_the_reference_state_dict_layout():
    """``MMInterleaved`` (H100) exposes the reference's parameter names for the parts whose reference classes import
    here (decoder + text head + glue): every key of the reference ``LlamaModel`` / ``TextDecoder`` layout exists."""
    import mm_interleaved_b200 as b200
    from tests.golden.make_golden import LLAMA_TINY
    ref_keys = {"mm_decoder." + k for k in _ref_layout("llama")}
    tiny_vt = dict(clip_config=b200.visual_tokenizer.CLIPVisionConfigLite(hidden_size=64, intermediate_size=128,
                                                                        num_hidden_layers=4, num_attention_heads=4,
                                                                        image_size=32, patch_size=8),
                   perceiver_config=dict(num_queries=3, hidden_size=48, encoder_hidden_size=64, num_hidden_layers=2,
                                         num_attention_heads=4, intermediate_size=96, cross_attention_frequency=1,
                                         qk_normalization=True), grid_size=4)
    try:
        model = b200.MMInterleaved(llm_config=dict(LLAMA_TINY, vocab_size=62), txt_vocab_size=64, seq_len=32,
                                   visual_tokenizer_config=tiny_vt, image_embed_dim=LLAMA_TINY["image_embed_dim"],
                                   cross_attention_frequency=2, spatial_shapes=LLAMA_TINY["spatial_shapes"])
    except Exception as e:                                                # tiny tokenizer dims unsupported on this build
        pytest.skip(f"tiny visual tokenizer config not constructible: {e}")
    keys = set(model.state_dict().keys())
    assert ref_keys <= keys, sorted(ref_keys - keys)[:5]
    for k in ("text_decoder.head.weight", "text_decoder.head.bias", "text_decoder.head_new.weight",
              "text_decoder.head_new.bias", "soi_token", "context_feat_proj.weight", "context_feat_proj.bias"):
        assert k in keys, k
    assert model.text_decoder.head.weight.shape[0] == 64 and model.text_decoder.head_new.weight.shape[0] == 2
    assert any(k.startswith("visual_tokenizer.encoder.") for k in keys)
