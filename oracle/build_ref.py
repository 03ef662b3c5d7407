"""oracle/build_ref.py -- compile the REFERENCE's own CUDA op as a GPU-side checker (oracle/_ref/).

TEST INFRASTRUCTURE ONLY.  Runs only where /root/reference exists (the build container); the resulting
oracle/_ref/MultiScaleDeformableAttention_ref*.so is git-ignored and travels to the GPU box with the snapshot.

The reference sources are compiled from where they lie (ops/src/vision.cpp, ops/src/cpu/ms_deform_attn_cpu.cpp,
ops/src/cuda/ms_deform_attn_cuda.cu + headers); nothing is copied into the repository.  They do not compile
against torch >= 2.x as shipped: `value.type()` is passed to AT_DISPATCH_FLOATING_TYPES_AND_HALF at
cuda/ms_deform_attn_cuda.cu:65 and :140 (DeprecatedTypeProperties -> ScalarType conversion was removed), so the
recipe compiles a scratch copy under /tmp with exactly those two tokens rewritten to `value.scalar_type()`
(SURVEY.md preamble); the kernels (ms_deform_im2col_cuda.cuh) are untouched.  The reference's own setup.py is not
used (it refuses to run without a visible GPU, ops/setup.py:36-47).
"""
from __future__ import annotations

import glob
import os
import re
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = "/root/reference/mm_interleaved/models/utils/ops/src"
OUT = os.path.join(HERE, "_ref")
NAME = "MultiScaleDeformableAttention_ref"


def main():
    if not os.path.isdir(REF_SRC):
        print("reference sources not present; nothing to build")
        return 0
    if glob.glob(os.path.join(OUT, NAME + "*.so")) and "--force" not in sys.argv:
        print("oracle/_ref already built")
        return 0
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="msda_ref_")
    shutil.copytree(REF_SRC, os.path.join(tmp, "src"))
    cu = os.path.join(tmp, "src", "cuda", "ms_deform_attn_cuda.cu")
    text = open(cu).read()
    patched, n = re.subn(r"AT_DISPATCH_FLOATING_TYPES_AND_HALF\(value\.type\(\)", "AT_DISPATCH_FLOATING_TYPES_AND_HALF(value.scalar_type()", text)
    assert n == 2, f"expected to patch 2 dispatch sites, found {n}"
    open(cu, "w").write(patched)
    vis = os.path.join(tmp, "src", "vision.cpp")
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    from torch.utils.cpp_extension import load
    srcs = [vis, os.path.join(tmp, "src", "cpu", "ms_deform_attn_cpu.cpp"), cu]
    load(name=NAME, sources=srcs, extra_include_paths=[os.path.join(tmp, "src")],
         extra_cflags=["-DWITH_CUDA", "-O2"],
         extra_cuda_cflags=["-DWITH_CUDA", "-gencode", "arch=compute_90a,code=sm_90a", "-DCUDA_HAS_FP16=1",
                            "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__"],
         build_directory=OUT, verbose="-v" in sys.argv, is_python_module=True)
    for f in glob.glob(os.path.join(OUT, "*")):
        if not f.endswith(".so"):
            os.remove(f)
    shutil.rmtree(tmp, ignore_errors=True)
    print("built", glob.glob(os.path.join(OUT, "*.so")))
    return 0


if __name__ == "__main__":
    sys.exit(main())
