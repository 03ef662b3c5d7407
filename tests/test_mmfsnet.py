"""MMFSNet (SD-UNet conditioning branch, decoders/sd_mmfs.py:154-272): CPU oracle pinned to the committed reference
outputs, and the H100 module against the same golden on the GPU (fp32: |err| <= 1e-3*|ref| + 1e-5*max|ref|)."""
import os

import numpy as np
import pytest
import torch

from oracle.sd_mmfs import mmfsnet_ref
from tests.golden.make_golden import MMFSNET_TINY, mmfsnet_inputs, mmfsnet_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mmfsnet_tiny.npz")


def _setup():
    import mm_interleaved_b200 as m
    net = m.MMFSNet(**MMFSNET_TINY)
    sd = mmfsnet_state_dict(net.state_dict())
    z = np.load(GOLDEN)
    assert abs(float(sum(v.double().sum() for v in sd.values())) - float(z["weight_checksum"])) < 1e-5
    net.load_state_dict(sd, strict=True)
    return net, sd, z


def test_oracle_matches_reference_golden():
    _, sd, z = _setup()
    sample, res, feats, mask = mmfsnet_inputs()
    out_sample, out_res = mmfsnet_ref(sd, sample, res, feats, mask, downsample_factor=8, n_down=4)
    assert (out_sample - torch.from_numpy(z["sample"])).abs().max() < 1e-5
    for i, r in enumerate(out_res):
        assert (r - torch.from_numpy(z[f"res{i}"])).abs().max() < 1e-5


@pytest.mark.gpu
def test_b200_module_matches_reference_golden():
    torch.backends.cuda.matmul.allow_tf32 = False
    net, _, z = _setup()
    net = net.cuda().eval()
    sample, res, feats, mask = mmfsnet_inputs()
    with torch.no_grad():
        out_sample, out_res = net(sample.cuda(), [r.cuda() for r in res], [f.cuda() for f in feats], mask.cuda())
        out2, _ = net(sample.cuda(), [r.cuda() for r in res], [f.cuda() for f in feats], mask.cuda())   # cached path
    for got, want in [(out_sample, z["sample"])] + [(r, z[f"res{i}"]) for i, r in enumerate(out_res)]:
        want = torch.from_numpy(want)
        err = (got.cpu() - want).abs()
        assert (err <= 1e-3 * want.abs() + 1e-5 * want.abs().max()).all(), err.max()   # abs floor relative to the tensor scale (~10)
    assert torch.equal(out2, out_sample)
