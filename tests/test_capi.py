"""CPU tests of the C-ABI boundary: the library loads without a GPU and exports every symbol
that include/mmfs_b200.h declares; argument validation returns the documented codes."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "mmfs_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mmfs_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol_at_abi_3():
    from mm_interleaved_b200 import _lib
    lib = _lib.lib()
    syms = header_symbols()
    assert len(syms) >= 7
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/mmfs_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature"
    assert lib.mmfs_abi_version() == 3


def test_msda_forward_argument_validation_without_gpu():
    from mm_interleaved_b200 import _lib
    lib = _lib.lib()
    # null pointers / bad dims are rejected before any CUDA call
    rc = lib.mmfs_msda_forward(None, None, None, None, None, None, 1, 4, 1, 8, 1, 1, 1, _lib.F32, 0, None)
    assert rc == _lib.EINVAL and b"null pointer" in lib.mmfs_last_error()
    rc = lib.mmfs_msda_forward(None, None, None, None, None, None, 1, 4, 1, 8, 0, 1, 1, _lib.F32, 0, None)
    assert rc == _lib.EINVAL
    rc = lib.mmfs_msda_forward(None, None, None, None, None, None, 1, 4, 1, 8, 1, 1, 1, 99, 0, None)
    assert rc == _lib.EINVAL and b"dtype" in lib.mmfs_last_error()
    # empty batch is a no-op success (the reference returns an empty tensor)
    rc = lib.mmfs_msda_forward(None, None, None, None, None, None, 0, 4, 1, 8, 1, 1, 1, _lib.F32, 0, None)
    assert rc == _lib.OK


def test_python_shim_mirrors_reference_errors():
    import MultiScaleDeformableAttention as MSDA
    from oracle import make_msda_inputs
    v, s, st, loc, a = make_msda_inputs(2, [(4, 4)], 2, 8, 3, 2)
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):   # ms_deform_attn.h:38
        MSDA.ms_deform_attn_forward(v, s, st, loc, a, 1)
    with pytest.raises(RuntimeError, match="contiguous"):                    # cu:29
        MSDA.ms_deform_attn_forward(v.transpose(1, 2), s, st, loc, a, 1)
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        MSDA.ms_deform_attn_backward(v, s, st, loc, a, torch.zeros(2, 3, 16), 1)


def test_no_product_import_of_oracle():
    """The product package must never import oracle/ (a CPU fallback voids parity claims)."""
    pkg = os.path.join(ROOT, "mm-interleaved_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f
    text = open(os.path.join(ROOT, "MultiScaleDeformableAttention", "__init__.py")).read()
    assert "oracle" not in text
