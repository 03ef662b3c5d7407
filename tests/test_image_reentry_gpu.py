"""ops.image_reentry (csrc/image_reentry_sm100.cu) against the reference's PIL host path (tests/golden/reentry.npz,
written by tests/golden/make_reentry.py): bit-identical on every case, run-to-run identical, other shapes refused."""
import os

import numpy as np
import pytest
import torch

from tests.golden.make_reentry import input_sha1, make_inputs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reentry.npz")
CASES = make_inputs()

pytestmark = pytest.mark.gpu


def _fixture(name):
    z = np.load(GOLDEN)
    images, R = CASES[name]
    assert input_sha1(images) == str(z[f"{name}/sha1"]), f"inputs of '{name}' do not reproduce"
    assert int(z[f"{name}/R"]) == R
    return torch.from_numpy(images), torch.from_numpy(z[f"{name}/u8"].astype(np.float32) / np.float32(255.0))


@pytest.mark.parametrize("name", sorted(CASES))
def test_bit_identical_to_pil(name):
    from mm_interleaved_b200 import ops
    images, ref = _fixture(name)
    out = ops.image_reentry(images.cuda(), ref.shape[-1]).cpu()
    assert out.shape == ref.shape
    diff = (out.view(torch.int32) != ref.view(torch.int32))
    assert not bool(diff.any()), f"{int(diff.sum())} of {diff.numel()} values differ, max |d| * 255 = " \
                                 f"{float((out - ref).abs().max()) * 255:.3f}"


def test_two_runs_and_out_slot_identical():
    from mm_interleaved_b200 import ops
    images, ref = _fixture("s512_noise")
    x = images.cuda()
    a = ops.image_reentry(x, 224)
    slots = torch.zeros((3, 3, 224, 224), device="cuda")
    b = ops.image_reentry(x, 224, out=slots[2:])
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert torch.equal(slots[2:].cpu().view(torch.int32), ref.view(torch.int32))
    assert not bool(slots[:2].any())


@pytest.mark.parametrize("shape", [(1, 3, 512, 256), (1, 4, 512, 512), (1, 1, 64, 64)])
def test_unsupported_shapes_raise(shape):
    from mm_interleaved_b200 import ops
    with pytest.raises(RuntimeError, match="unsupported"):
        ops.image_reentry(torch.rand(shape, device="cuda"), 224)


def test_bad_arguments_raise():
    from mm_interleaved_b200 import ops
    with pytest.raises(RuntimeError):
        ops.image_reentry(torch.rand((1, 3, 64, 64), device="cuda", dtype=torch.float16), 32)
    with pytest.raises(RuntimeError):
        ops.image_reentry(torch.rand((1, 3, 64, 64), device="cuda"), 32, out=torch.empty((1, 3, 16, 16), device="cuda"))
