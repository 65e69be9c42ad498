"""Compile the reference's own CPU attention (flash_attention_c) UNMODIFIED into oracle/_ref/.

Sources are compiled where they lie in the reference checkout named by TFA_REFERENCE (never copied into this repo):
    flash_attention_c/csrc/attn.cpp   naive_attn / flash_attn (OpenMP)
    flash_attention_c/csrc/ops.cu     pybind glue (PYBIND11_MODULE(_kernels))
The reference's own CMake build is not run; this is the short recipe SURVEY.md section 8c verified:
torch.utils.cpp_extension.load with -O3 -fopenmp.  Output: oracle/_ref/_kernels.so (git-ignored); where the
reference's sources are absent, an oracle/_ref built elsewhere is used as it is, and without one the tests that call
it skip.
"""
from __future__ import annotations

import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("TFA_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "_ref")


def build_ref(force: bool = False, verbose: bool = False):
    src_dir = os.path.join(REF, "flash_attention_c", "csrc")
    srcs = [os.path.join(src_dir, "attn.cpp"), os.path.join(src_dir, "ops.cu")]
    target = os.path.join(OUT, "_kernels.so")
    if not all(os.path.exists(s) for s in srcs):
        return target if os.path.exists(target) else None      # no sources here: use a prebuilt file, if any
    if os.path.exists(target) and not force:
        return target
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils.cpp_extension import load

    build_dir = os.path.join(OUT, "_build")
    os.makedirs(build_dir, exist_ok=True)
    load(name="_kernels", sources=srcs, extra_cflags=["-O3", "-fopenmp"],
         extra_ldflags=["-L/usr/lib/gcc/x86_64-linux-gnu/13", "-lgomp"], with_cuda=True,
         build_directory=build_dir, verbose=verbose, is_python_module=False)
    built = os.path.join(build_dir, "_kernels.so")
    shutil.copy2(built, target)
    return target


if __name__ == "__main__":
    print(build_ref(force="--force" in sys.argv, verbose=True))
