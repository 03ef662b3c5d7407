"""CPU tests of the ViT-Adapter training path: the argument checks of its two backward kernels
(``mmfs_quick_gelu_backward``, ``mmfs_resize_bilinear_backward``) and of their Python wrappers (every malformed or
unsupported call is rejected with MMFS_EINVAL / MMFS_EUNSUPPORTED and a message before any CUDA call), the guard of the
raw MSDA forward under autograd, ``VisualTokenizer.freeze_like_reference()`` against the trainable set of the
reference's own code (tests/golden/adapter_grad_tiny.npz), and the generator of that fixture."""
import os

import numpy as np
import pytest
import torch

GOOD = 0x1000            # stands for a valid device pointer; no call below gets far enough to dereference it
BF16, F16, F32 = 2, 1, 0
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gelu(**over):
    from mm_interleaved_b200 import _lib
    a = dict(h=GOOD, dy=GOOD, dh=GOOD, n=4 * 257 * 4096, dtype=BF16)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_quick_gelu_backward(a["h"], a["dy"], a["dh"], a["n"], a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


def _resize(**over):
    from mm_interleaved_b200 import _lib
    a = dict(dy=GOOD, dx=GOOD, B=4, C=1024, Hin=16, Win=16, Hout=64, Wout=64, bs=64 * 64 * 1024, cs=1, ps=1024,
             sh=0.25, sw=0.25, dtype=BF16)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_resize_bilinear_backward(a["dy"], a["dx"], a["B"], a["C"], a["Hin"], a["Win"], a["Hout"], a["Wout"],
                                           a["bs"], a["cs"], a["ps"], a["sh"], a["sw"], a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


@pytest.mark.parametrize("over,code,text", [
    (dict(h=None), "EINVAL", "null pointer"), (dict(dy=None), "EINVAL", "null pointer"),
    (dict(dh=None), "EINVAL", "null pointer"), (dict(n=-1), "EINVAL", "bad shape"),
    (dict(dtype=F32), "EUNSUPPORTED", "bf16"), (dict(dtype=3), "EUNSUPPORTED", "bf16"),
    (dict(dtype=7), "EUNSUPPORTED", "bf16"), (dict(h=GOOD + 2), "EUNSUPPORTED", "aligned"),
    (dict(dh=GOOD + 8), "EUNSUPPORTED", "aligned"),
])
def test_quick_gelu_backward_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _gelu(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


def test_quick_gelu_backward_empty_call_returns_before_the_pointers():
    from mm_interleaved_b200 import _lib
    assert _gelu(n=0, h=None)[0] == _lib.OK


@pytest.mark.parametrize("over,code,text", [
    (dict(dy=None), "EINVAL", "null pointer"), (dict(dx=None), "EINVAL", "null pointer"),
    (dict(B=-1), "EINVAL", "bad shape"), (dict(C=0), "EINVAL", "bad shape"), (dict(Hin=0), "EINVAL", "bad shape"),
    (dict(Wout=0), "EINVAL", "bad shape"), (dict(sh=0.0), "EINVAL", "bad shape"), (dict(sw=-2.0), "EINVAL", "bad shape"),
    (dict(dtype=F32), "EUNSUPPORTED", "bf16"), (dict(dtype=3), "EUNSUPPORTED", "bf16"),
    (dict(C=1020), "EUNSUPPORTED", "C % 8"), (dict(dx=GOOD + 4), "EUNSUPPORTED", "aligned"),
])
def test_resize_bilinear_backward_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _resize(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


def test_resize_bilinear_backward_empty_batch_returns_before_the_pointers():
    from mm_interleaved_b200 import _lib
    assert _resize(B=0, dy=None, dx=None)[0] == _lib.OK


def test_wrappers_refuse_bad_tensors():
    """Shapes, dtypes and devices are checked before the library sees the call (CPU tensors fail the first check)."""
    from mm_interleaved_b200 import ops
    with pytest.raises(RuntimeError, match="quick_gelu_backward"):
        ops.quick_gelu_backward(torch.zeros(4, 64), torch.zeros(4, 64))
    with pytest.raises(RuntimeError, match="resize_bilinear_backward"):
        ops.resize_bilinear_backward(torch.zeros(1, 8, 16, 16), (4, 4), 4)
    with pytest.raises(RuntimeError, match="resize_bilinear_backward"):
        ops.resize_bilinear_backward(torch.zeros(1, 8, 16), (4, 4), 4)


def test_kernels_refuse_to_run_under_autograd():
    """Neither the new wrappers nor the raw MSDA forward may run where autograd would drop a gradient."""
    from mm_interleaved_b200 import msda, ops
    h = torch.zeros(4, 64, requires_grad=True)
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.quick_gelu_backward(h, torch.zeros(4, 64))
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.resize_bilinear_backward(torch.zeros(1, 8, 16, 16, requires_grad=True), (4, 4), 4)
    value = torch.zeros(1, 16, 2, 32, requires_grad=True)
    ss, st = torch.tensor([[4, 4]]), torch.tensor([0])
    loc, attn = torch.zeros(1, 3, 2, 1, 4, 2), torch.zeros(1, 3, 2, 1, 4)
    with pytest.raises(RuntimeError, match="inference-only"):
        msda.ms_deform_attn_forward(value, ss, st, loc, attn, 1)


def _tiny_tokenizer():
    from mm_interleaved_b200 import visual_tokenizer as vt
    from tests.golden.make_adapter_grad import ADAPTER_GRAD_TINY as c
    return vt.VisualTokenizer(clip_config=vt.CLIPVisionConfigLite(**c["clip"]), perceiver_config=dict(c["perceiver"]),
                              llm_hidden_size=c["llm_hidden_size"], grid_size=c["grid_size"])


def test_freeze_like_reference_matches_the_reference_trainable_set():
    """The reference's own clip_vit_adapter_hf(freeze=False, freeze_vit=True) inside its VisualTokenizer decides which
    tensors train; the names are this repository's too (its checkpoints load unchanged)."""
    z = np.load(os.path.join(GOLDEN, "adapter_grad_tiny.npz"))
    tok = _tiny_tokenizer()
    tok.requires_grad_(True)
    assert tok.freeze_like_reference() is tok
    got = sorted(n for n, p in tok.named_parameters() if p.requires_grad)
    assert got == [str(n) for n in z["trainable"]]
    assert not tok.pos_embed.requires_grad
    assert any(n.startswith("encoder.vision_model.adapter_spm.") for n in got)
    assert not any(n.startswith("encoder.vision_model.encoder.") or ".embeddings." in n for n in got)
    tok.requires_grad_(False)
    assert sorted(n for n, p in tok.freeze_like_reference().named_parameters() if p.requires_grad) == got


def test_trainable_clip_weights_still_raise_in_mm_interleaved():
    """Only the adapter (and head) may train: a trainable CLIP weight still raises up front, with the recipe."""
    import mm_interleaved_b200 as m
    from tests.golden.make_golden import LLAMA_TINY
    vt_cfg = dict(clip_config=m.visual_tokenizer.CLIPVisionConfigLite(hidden_size=64, intermediate_size=64, num_hidden_layers=4,
                                                                     num_attention_heads=2, image_size=28, patch_size=14),
                  perceiver_config=dict(num_queries=2, hidden_size=64, encoder_hidden_size=64, cross_attention_frequency=2,
                                        num_hidden_layers=2, num_attention_heads=2, intermediate_size=64,
                                        qk_normalization=True), grid_size=2)
    st = dict(bos_token_id=1, eos_token_id=2, pad_token_id=0, soi_token_id=62, image_token_id=63)
    model = m.MMInterleaved(llm_config=dict(LLAMA_TINY, vocab_size=62), txt_vocab_size=64, seq_len=32, special_token_dict=st,
                            visual_tokenizer_config=vt_cfg, image_embed_dim=LLAMA_TINY["image_embed_dim"],
                            cross_attention_frequency=2, spatial_shapes=LLAMA_TINY["spatial_shapes"]).freeze_like_reference()
    ids = torch.ones(1, 4, dtype=torch.long)
    with pytest.raises(RuntimeError, match="the visual tokenizer has no backward.*freeze_like_reference"):
        model(text_ids=ids, attention_mask=torch.ones_like(ids))


def test_golden_generator_reproduces_the_fixture(tmp_path):
    """tests/golden/make_adapter_grad.py runs the reference's own tokenizer to completion and rewrites the fixture."""
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("the reference tree is not installed here")
    from tests.golden import make_adapter_grad
    path = tmp_path / "adapter_grad_tiny.npz"
    make_adapter_grad.main(str(path))
    new, old = np.load(path), np.load(os.path.join(GOLDEN, "adapter_grad_tiny.npz"))
    assert sorted(new.files) == sorted(old.files)
    assert list(new["trainable"]) == list(old["trainable"])
    for k in new.files:
        if k.startswith(("grad/", "out/")):
            np.testing.assert_allclose(new[k], old[k], rtol=1e-5, atol=1e-6 * float(np.abs(old[k]).max()), err_msg=k)
