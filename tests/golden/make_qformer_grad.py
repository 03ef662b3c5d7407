"""Generate tests/golden/qformer_grad_tiny.npz from the UNMODIFIED reference's Q-Former, executed in the build container
through oracle/ref_loader.load_visual() (the shims of make_golden.make_tokenizer: transformers 5.x Q-Former glue standing
in for 4.31).

    python tests/golden/make_qformer_grad.py

The Q-Former (decoders/perceiver.py + utils/monkey_patch/blip2_qknorm_monkey_patch.py) at head dim 64, float64, dropout
0: the output and the gradients of a fixed seeded projection of it with respect to every parameter and to
encoder_hidden_states, with and without a key-padding mask.  To keep the fixture small, every tensor of more than
SAMPLE entries is stored as the fixed sample ``sample_index(numel)`` of its flattened entries, in fp32 (the 16-bit checks
against it are three orders looser than fp32).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.golden.make_golden import ref_loader, tokenizer_state_dict  # noqa: E402

QFORMER_GRAD_TINY = dict(num_queries=8, hidden_size=128, encoder_hidden_size=96, num_hidden_layers=2, num_attention_heads=2,
                         cross_attention_frequency=2, intermediate_size=256, qk_normalization=True)
WEIGHT_SEED = 929
SAMPLE = 512                  # entries kept of a larger tensor


def sample_index(numel):
    """The flattened entries kept of a tensor with ``numel`` entries: all of them up to SAMPLE, else a fixed sorted
    sample of SAMPLE."""
    if numel <= SAMPLE:
        return torch.arange(numel)
    return torch.randperm(numel, generator=torch.Generator().manual_seed(numel))[:SAMPLE].sort().values


def sample(t):
    return t.reshape(-1)[sample_index(t.numel())]


def qformer_grad_inputs(seed=53):
    """(encoder_hidden_states (2, 17, 96), key mask (2, 17) with the second entry's last 6 keys padded, output projection
    (2, 8, 128)), float64."""
    g = torch.Generator().manual_seed(seed)
    c = QFORMER_GRAD_TINY
    enc = torch.randn((2, 17, c["encoder_hidden_size"]), generator=g, dtype=torch.float64)
    mask = torch.ones((2, 17), dtype=torch.long)
    mask[1, 11:] = 0
    proj = torch.randn((2, c["num_queries"], c["hidden_size"]), generator=g, dtype=torch.float64)
    return enc, mask, proj


def main():
    ns = ref_loader.load_visual()
    per = ns.perceiver.PerceiverResampler(**QFORMER_GRAD_TINY, gradient_checkpointing=False, hidden_dropout_prob=0.0,
                                          attention_probs_dropout_prob=0.0).eval()
    sd = tokenizer_state_dict(per.state_dict(), seed=WEIGHT_SEED)
    per.load_state_dict(sd)
    per = per.double()
    enc, mask, proj = qformer_grad_inputs()
    out = {}
    for tag, m in (("masked", mask), ("unmasked", None)):
        per.zero_grad(set_to_none=True)
        e = enc.clone().requires_grad_(True)
        o = per(encoder_hidden_states=e, encoder_attention_mask=m, return_dict=False)[0]
        (o * proj).sum().backward()
        out[f"{tag}/out"] = sample(o.detach())
        out[f"{tag}/encoder_hidden_states"] = sample(e.grad)
        for n, prm in per.named_parameters():
            out[f"{tag}/{n}"] = sample(prm.grad)
    path = os.path.join(HERE, "qformer_grad_tiny.npz")
    np.savez_compressed(path, **{k: v.numpy().astype(np.float32) for k, v in out.items()}, keys=np.array(sorted(sd.keys())),
                        checksum=np.array(float(sum(v.double().sum() for v in sd.values()))))
    print(f"{path}: {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    torch.manual_seed(0)
    main()
