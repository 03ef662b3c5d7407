"""Generate tests/golden/adapter_grad_tiny.npz from the UNMODIFIED reference's visual tokenizer, executed in the build
container through oracle/ref_loader.load_visual() (the shims of make_golden.make_tokenizer: transformers 5.x CLIP /
Q-Former glue standing in for 4.31).

    python tests/golden/make_adapter_grad.py

The reference's ``VisualTokenizer`` (CLIP ViT + ViT-Adapter + qk-norm Q-Former) in float64 at a tiny size with the real
per-head shapes: CLIP hidden 128 over 2 heads (head dim 64) and 24 layers (the adapter's hard-coded interaction indexes),
112^2 images (8 x 8 patches, T = 65 tokens: more than one 64-key attention tile), MSDA head size 128 * 0.5 / 2 = 32, a
2-layer Q-Former at head dim 64, 2 images.  The trainable set is the one the reference's own
``clip_vit_adapter_hf(freeze=False, freeze_vit=True)`` leaves (with ``from_pretrained`` returning the tiny model): every
``vision_model.adapter*`` parameter, the head, not ``pos_embed``.  Stored: the sorted trainable names, the outputs, and
the gradient of every trainable tensor of a seeded projection of ALL outputs (vis_embed, image_embeds and the four
multi-scale maps, so every output route and all three resizes carry gradient), each as the fixed sample
``sample_index(numel)`` of make_qformer_grad.py, in fp32.  Injector ``gamma`` is 0.7 (zero-initialised in the
reference), so the injectors get gradient.  For per-stage comparisons it also stores, sampled the same way, the gradient
arriving at the spatial prior module's four outputs (``stage/c1`` .. ``stage/c4``, as ``SPM_STAGES`` names them).
"""
from __future__ import annotations

import functools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.golden.make_golden import ref_loader, tokenizer_state_dict  # noqa: E402
from tests.golden.make_qformer_grad import sample  # noqa: E402

ADAPTER_GRAD_TINY = dict(clip=dict(hidden_size=128, intermediate_size=256, num_hidden_layers=24, num_attention_heads=2,
                                   image_size=112, patch_size=14),
                         perceiver=dict(num_queries=8, hidden_size=128, encoder_hidden_size=128, cross_attention_frequency=2,
                                        num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                                        qk_normalization=True),
                         llm_hidden_size=96, grid_size=8)
WEIGHT_SEED = 939
OUTPUTS = ("vis_embed", "image_embeds", "ms0", "ms1", "ms2", "ms3")
SPM_STAGES = ("c1", "c2", "c3", "c4")


def retain_stage_grads(spm):
    """Forward hook on a spatial prior module: keeps the gradients of its four outputs.  Returns the dict it fills
    (stage name -> output tensor, whose ``.grad`` is set by the backward)."""
    kept = {}

    def hook(_mod, _inp, out):
        for name, t in zip(SPM_STAGES, out):
            if t.requires_grad:
                t.retain_grad()
                kept[name] = t
    spm.register_forward_hook(hook)
    return kept


def flat_outputs(out):
    """{name: tensor} of a tokenizer output dict, in OUTPUTS order."""
    d = dict(vis_embed=out["vis_embed"], image_embeds=out["image_embeds"])
    d.update({f"ms{i}": f for i, f in enumerate(out["multiscale_features"])})
    return d


def adapter_grad_inputs(seed=59):
    """(images (2, 3, 112, 112) in [0, 1], {output name: projection of that output's shape}), float64."""
    g = torch.Generator().manual_seed(seed)
    c = ADAPTER_GRAD_TINY
    s, d, n = c["clip"]["image_size"], c["clip"]["hidden_size"], c["clip"]["image_size"] // c["clip"]["patch_size"]
    images = torch.rand((2, 3, s, s), generator=g, dtype=torch.float64)
    shapes = dict(vis_embed=(2, c["perceiver"]["num_queries"], c["llm_hidden_size"]), image_embeds=(2, n * n, d),
                  ms0=(2, d, 4 * n, 4 * n), ms1=(2, d, 2 * n, 2 * n), ms2=(2, d, n, n), ms3=(2, d, n // 2, n // 2))
    proj = {k: torch.randn(shapes[k], generator=g, dtype=torch.float64) for k in OUTPUTS}
    return images, proj


def main(path=os.path.join(HERE, "adapter_grad_tiny.npz")):
    from transformers import CLIPVisionConfig
    ns = ref_loader.load_visual()
    c = ADAPTER_GRAD_TINY
    cfg = CLIPVisionConfig(**c["clip"], hidden_act="quick_gelu", layer_norm_eps=1e-5)
    cfg._attn_implementation = "eager"
    # clip_vit_adapter_hf (vit_adapter_hf.py:231-254) as the reference calls it, with from_pretrained giving the tiny model
    ns.vit_adapter.CLIPVisionAdapterModel.from_pretrained = classmethod(lambda cls, *a, **k: cls(cfg))
    ns.visual_tokenizer.clip_vit_adapter_hf = functools.partial(
        ns.vit_adapter.clip_vit_adapter_hf, image_size=c["clip"]["image_size"], freeze=False, freeze_vit=True,
        gradient_checkpointing=False)
    pc = ref_loader.AttrDict(c["perceiver"], gradient_checkpointing=False, hidden_dropout_prob=0.0,
                             attention_probs_dropout_prob=0.0)
    tok = ns.visual_tokenizer.VisualTokenizer(encoder_model_path="", perceiver_config=pc, llm_hidden_size=c["llm_hidden_size"],
                                              grid_size=c["grid_size"]).eval()
    sd = tokenizer_state_dict(tok.state_dict(), seed=WEIGHT_SEED)
    tok.load_state_dict(sd)
    tok = tok.double()
    trainable = sorted(n for n, p in tok.named_parameters() if p.requires_grad)
    images, proj = adapter_grad_inputs()
    stages = retain_stage_grads(tok.encoder.vision_model.adapter_spm)
    outs = flat_outputs(tok(images))
    sum((outs[k] * proj[k]).sum() for k in OUTPUTS).backward()
    arrays = {f"out/{k}": sample(outs[k].detach()) for k in OUTPUTS}
    arrays.update({f"stage/{k}": sample(stages[k].grad) for k in SPM_STAGES})
    params = dict(tok.named_parameters())
    for n in trainable:
        arrays[f"grad/{n}"] = sample(params[n].grad)
    np.savez_compressed(path, **{k: v.numpy().astype(np.float32) for k, v in arrays.items()},
                        trainable=np.array(trainable), keys=np.array(sorted(sd.keys())),
                        checksum=np.array(float(sum(v.double().sum() for v in sd.values()))))
    print(f"{path}: {os.path.getsize(path) / 1024:.0f} KiB, {len(trainable)} trainable tensors")


if __name__ == "__main__":
    torch.manual_seed(0)
    main()
