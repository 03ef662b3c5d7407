"""oracle/ref_cuda.py -- load the reference's own CUDA op (built by oracle/build_ref.py into oracle/_ref/).

TEST INFRASTRUCTURE ONLY.  Gives the GPU tests and the sweep tool the REAL reference kernel on the H100:
``ms_deform_attn_forward(value, shapes, level_start_index, sampling_loc, attn_weight, im2col_step)`` exactly as
ops/src/vision.cpp:13-16 exposes it (fp64 / fp32 / fp16; no bf16 dispatch, cu:65)."""
from __future__ import annotations

import glob
import importlib.machinery
import importlib.util
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_mod = None


def available() -> bool:
    return bool(glob.glob(os.path.join(_HERE, "_ref", "MultiScaleDeformableAttention_ref*.so")))


def load():
    global _mod
    if _mod is None:
        import torch  # noqa: F401  (libtorch must be loaded first)
        path = glob.glob(os.path.join(_HERE, "_ref", "MultiScaleDeformableAttention_ref*.so"))[0]
        loader = importlib.machinery.ExtensionFileLoader("MultiScaleDeformableAttention_ref", path)
        spec = importlib.util.spec_from_loader("MultiScaleDeformableAttention_ref", loader)
        _mod = importlib.util.module_from_spec(spec)
        loader.exec_module(_mod)
    return _mod
