"""Generate tests/golden/reentry.npz: the reference's own host path for a generated image re-entering the context,
``update_image`` of inference.py -- ``tensor_to_pil`` (utils/clip_sim_score.py) and ``create_transform("numpy", R)``
(custom_datasets/utils.py: ``center_crop_arr`` with PIL's BOX and BICUBIC resizes, then ``/ 255``) -- on seeded images.

    python tests/golden/make_reentry.py

The two reference functions are compiled from the reference's files as they are (their modules import training-only
dependencies, so only the function definitions are taken).  The inputs are rebuilt from ``make_inputs()`` (seeded
numpy) and checked against the stored SHA-1; the outputs are stored as the uint8 values u with the output = float32(u)
/ 255.  Cases: the shipped 512 -> 224 (one BOX halving, then bicubic 256 -> 224), sizes that take zero (224, 300, 160:
identity, bicubic down, bicubic up), one (448) and two (1024) halvings, values at the quantisation boundaries
(k / 255 and (k - 0.5) / 255, +-1 ulp) and outside [0, 1], constant images and single-pixel impulses (the filters'
support).
"""
from __future__ import annotations

import ast
import hashlib
import math
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("MMI_REFERENCE_ROOT", "/root/reference")


def _boundary_values():
    k = np.arange(256, dtype=np.float64)
    base = np.concatenate([k / 255.0, (k - 0.5) / 255.0, (k + 0.5) / 255.0]).astype(np.float32)
    up, down = np.nextafter(base, np.float32(np.inf)), np.nextafter(base, np.float32(-np.inf))
    extra = np.array([-1.0, -0.25, -1e-7, 0.0, 1.0, 1.0 + 1e-7, 1.25, 3.0], dtype=np.float32)
    return np.concatenate([base, up, down, extra])


def make_inputs():
    """name -> (images (N, 3, S, S) float32, R)."""
    rng = np.random.default_rng(20261017)
    cases = {}

    def noise(n, s, lo=-0.05, hi=1.05):
        return rng.uniform(lo, hi, size=(n, 3, s, s)).astype(np.float32)

    def smooth(n, s):
        y, x = np.meshgrid(np.linspace(0, 1, s), np.linspace(0, 1, s), indexing="ij")
        ph = rng.uniform(0, 2 * np.pi, size=(n, 3, 1, 1))
        img = 0.5 + 0.45 * np.sin(7 * x[None, None] + 5 * y[None, None] + ph)
        return (img + rng.normal(0, 0.02, size=img.shape)).astype(np.float32)

    vals = _boundary_values()
    cases["s512_noise"] = (noise(1, 512), 224)
    cases["s512_smooth"] = (smooth(1, 512), 224)
    cases["s512_boundary"] = (rng.choice(vals, size=(1, 3, 512, 512)).astype(np.float32), 224)
    flat = np.resize(vals, 3 * 224 * 224).astype(np.float32)
    cases["s224_boundary"] = (flat.reshape(1, 3, 224, 224), 224)
    cases["s448_smooth"] = (smooth(1, 448), 224)
    cases["s1024_smooth"] = (smooth(1, 1024), 224)
    cases["s300_smooth"] = (smooth(1, 300), 224)
    cases["s160_smooth"] = (smooth(1, 160), 224)
    const = np.stack([np.full((3, 512, 512), v, dtype=np.float32) for v in (0.0, 0.3, 0.5, 1.0, 7.0 / 255.0)])
    cases["s512_const"] = (const, 224)
    imp = np.zeros((2, 3, 512, 512), dtype=np.float32)
    for (y, x) in ((0, 0), (1, 511), (255, 256), (256, 255), (100, 3), (511, 300), (300, 508), (17, 17)):
        imp[0, :, y, x] = 1.0
    imp[1] += 1.0
    for (y, x) in ((0, 511), (2, 2), (128, 129), (509, 0), (400, 401)):
        imp[1, :, y, x] = 0.0
    cases["s512_impulse"] = (imp, 224)
    imp2 = np.zeros((1, 3, 256, 256), dtype=np.float32)
    for (y, x) in ((0, 0), (5, 250), (128, 128), (255, 1), (200, 64)):
        imp2[0, :, y, x] = 1.0
    cases["s256_impulse"] = (imp2, 224)
    cases["s97_odd"] = (noise(1, 97), 24)                    # odd sizes: 97 -> 48 (BOX, scale 97/48) -> 24 (BOX)
    return cases


def input_sha1(images: np.ndarray) -> str:
    return hashlib.sha1(np.ascontiguousarray(images).tobytes()).hexdigest()


def reference_functions():
    """``tensor_to_pil`` and ``create_transform`` compiled from the reference's own source files."""
    import torch
    from PIL import Image
    ns = {"np": np, "Image": Image, "math": math, "random": random, "torch": torch, "transforms": None}
    pkg = os.path.join(REF_ROOT, "mm_interleaved")
    for rel, names in (("utils/clip_sim_score.py", {"tensor_to_pil"}),
                       ("custom_datasets/utils.py", {"transform_numpy", "center_crop_arr", "random_crop_arr",
                                                     "create_transform"})):
        path = os.path.join(pkg, rel)
        tree = ast.parse(open(path).read(), path)
        body = [n for n in tree.body if getattr(n, "name", None) in names]
        assert {n.name for n in body} == names, f"{path}: {names - {n.name for n in body}} not found"
        exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns["tensor_to_pil"], ns["create_transform"]


def main():
    import torch
    tensor_to_pil, create_transform = reference_functions()
    out = {}
    for name, (images, R) in make_inputs().items():
        transform = create_transform("numpy", R)
        us = []
        for img in images:                                       # update_image: one image per call
            arr = transform(tensor_to_pil(torch.from_numpy(img)[None])[0])
            u = np.rint(arr * 255.0).astype(np.uint8)
            assert np.array_equal((u.astype(np.float32) / np.float32(255.0)), arr), name   # arr == float32(u) / 255
            us.append(u)
        out[f"{name}/u8"] = np.stack(us)
        out[f"{name}/sha1"] = np.array(input_sha1(images))
        out[f"{name}/R"] = np.array(R)
    path = os.path.join(HERE, "reentry.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    sys.exit(main())
