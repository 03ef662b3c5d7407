"""Generate tests/golden/mmfsnet_grad_tiny.npz from the UNMODIFIED reference's ``MMFSNet`` (decoders/sd_mmfs.py), executed
in the build container through oracle/ref_loader.load() (the MSDA gather is the reference's own PyTorch core,
func.py:47-67).

    python tests/golden/make_mmfsnet_grad.py

The reference's MMFSNet at the ``MMFSNET_TINY`` size of make_golden.py (feature width 64, block channels (32, 64), one
layer per block, downsample factor 8; attention width 1024 over 16 heads, so the MSDA head size is 64 as in SD) with
make_golden's seeded weights -- the zero-initialised 1x1 ``conv`` of every block scaled up, so that the hook's
parameters get gradient -- in float64, on ``mmfsnet_inputs()``.  Loss: a seeded projection of both outputs (the new
mid-block sample and the four new skip tensors).  Stored, in fp32: the outputs, the gradient arriving at the inputs
(sample, the four skips, the four feature maps) and the gradient of every trainable parameter, each as the fixed sample
``sample_index(numel)`` of make_qformer_grad.py; the sorted trainable names.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.golden.make_golden import MMFSNET_TINY, mmfsnet_inputs, mmfsnet_state_dict, ref_loader  # noqa: E402
from tests.golden.make_qformer_grad import sample  # noqa: E402


def mmfsnet_grad_inputs(seed=71):
    """(sample, skips, features, mask) of make_golden.mmfsnet_inputs() in float64, and the output projections
    (one for the new sample, one per new skip)."""
    s, res, feats, mask = mmfsnet_inputs()
    g = torch.Generator().manual_seed(seed)
    proj = [torch.randn(s.shape, generator=g, dtype=torch.float64)] + \
        [torch.randn(r.shape, generator=g, dtype=torch.float64) for r in res]
    return s.double(), [r.double() for r in res], [f.double() for f in feats], mask.double(), proj


def input_names(n_res, n_feats):
    return ["sample"] + [f"res{i}" for i in range(n_res)] + [f"feat{i}" for i in range(n_feats)]


def main(path=os.path.join(HERE, "mmfsnet_grad_tiny.npz")):
    ns = ref_loader.load()
    net = ns.sd_mmfs.MMFSNet(**MMFSNET_TINY).eval()
    sd = mmfsnet_state_dict(net.state_dict())
    net.load_state_dict(sd)
    net = net.double()
    trainable = sorted(n for n, p in net.named_parameters() if p.requires_grad)
    s, res, feats, mask, proj = mmfsnet_grad_inputs()
    inputs = [s, *res, *feats]
    for t in inputs:
        t.requires_grad_(True)
    out_sample, out_res = net(s, res, feats, mask)
    outs = [out_sample, *out_res]
    sum((o * p).sum() for o, p in zip(outs, proj)).backward()
    arrays = {f"out/{i}": sample(o.detach()) for i, o in enumerate(outs)}
    for name, t in zip(input_names(len(res), len(feats)), inputs):
        arrays[f"input_grad/{name}"] = sample(t.grad)
    params = dict(net.named_parameters())
    for n in trainable:
        arrays[f"grad/{n}"] = sample(params[n].grad)
    np.savez_compressed(path, **{k: v.numpy().astype(np.float32) for k, v in arrays.items()},
                        trainable=np.array(trainable),
                        checksum=np.array(float(sum(v.double().sum() for v in sd.values()))))
    print(f"{path}: {os.path.getsize(path) / 1024:.0f} KiB, {len(trainable)} trainable tensors")


if __name__ == "__main__":
    torch.manual_seed(0)
    main()
