"""Compile the UNMODIFIED reference rotation kernel into oracle/_ref/ (test infrastructure).

    python oracle/build_ref.py

Sources are compiled where they lie (REF: rotation.cu, rotation.cuh, pybind.cpp) -- nothing is copied into this
repository.  The recipe is ours (torch's cpp_extension driving nvcc/ninja directly), with the compiler flags the
reference's own loader passes (paroquant/kernels/cuda/__init__.py:30-41), for sm_90a.  Output:
oracle/_ref/paroquant_rotation.so (git-ignored), which tools/ref_gpu.py loads with torch.ops.load_library in a
separate process (it registers the same `rotation::rotate` op name as our own provider) to produce the golden data
under tests/golden/ and the same-GPU baseline of bench.py.

The GEMM half of the reference path is vLLM's Marlin, taken from the installed vllm wheel.
"""
from __future__ import annotations

import os
import sys
from pathlib import Path

REF = Path("/root/reference/paroquant/kernels/cuda")
OUT = Path(__file__).resolve().parent / "_ref"


def build() -> Path | None:
    so = OUT / "paroquant_rotation.so"
    if so.exists():
        return so
    if not REF.exists():
        return None  # GPU box: only the prebuilt file travels
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    from torch.utils.cpp_extension import load

    OUT.mkdir(exist_ok=True)
    load(name="paroquant_rotation", sources=[str(REF / "pybind.cpp"), str(REF / "rotation.cu")],
         build_directory=str(OUT), is_python_module=False,
         extra_cuda_cflags=["-O3", "-std=c++17", "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
                            "-U__CUDA_NO_BFLOAT16_OPERATORS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
                            "--expt-relaxed-constexpr", "--expt-extended-lambda", "--use_fast_math"],
         extra_cflags=["-O2", "-std=c++17"], verbose=False)
    return so if so.exists() else None


if __name__ == "__main__":
    print(build())
