"""Build the sm_90a (H100) extension in-tree.  ``python -m neuronx_distributed_b200.ops.build``

Uses ``torch.utils.cpp_extension.load`` with explicit ``-gencode arch=compute_90a,code=sm_90a``
(bypassing torch's arch list; nvcc cross-compiles without a GPU) and ``-lineinfo`` so ncu source
pages map to our code."""
from __future__ import annotations

import os
import sys
from pathlib import Path

from ._ext import BUILD_DIR, EXT_NAME, PKG_DIR

CSRC = PKG_DIR.parent / "csrc"


def sources():
    return sorted(str(p) for p in list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")))


def build(verbose: bool = False) -> Path:
    from torch.utils import cpp_extension

    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")  # only used for a sanity print; real arch below
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 4))
    cuda_flags = [
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-lineinfo", "-O3", "-std=c++17",
        "--expt-relaxed-constexpr", "--use_fast_math",
        "-Xptxas", "-v",
        "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
        "-U__CUDA_NO_BFLOAT16_CONVERSIONS__", "-U__CUDA_NO_HALF2_OPERATORS__",
    ]
    cpp_extension.load(
        name=EXT_NAME,
        sources=sources(),
        extra_cflags=["-O3", "-std=c++17"],
        extra_cuda_cflags=cuda_flags,
        extra_ldflags=["-lcuda"] if _has_libcuda() else [],
        extra_include_paths=[str(CSRC)],
        build_directory=str(BUILD_DIR),
        verbose=verbose,
        is_python_module=True,
        with_cuda=True,
    )
    so = BUILD_DIR / f"{EXT_NAME}.so"
    assert so.exists(), f"build did not produce {so}"
    return so


def _has_libcuda() -> bool:
    return False  # driver entry points are resolved at runtime via cudaGetDriverEntryPoint


if __name__ == "__main__":
    p = build(verbose="-v" in sys.argv)
    print(p)
