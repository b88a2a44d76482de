"""Python front-ends of the hand-written sm_90a kernels (``csrc/``).

Every op has (a) the CUDA path through the in-tree extension and (b) a plain PyTorch fp32
reference used on CPU and as the numerics oracle in tests.  On a GPU box the CUDA path is
mandatory (see ``_ext.use_cuda``).
"""
from . import _ext  # noqa: F401
from . import act, attention, cross_entropy, gemm, gemm_mx, moe_tkg, norm, nvls, optim, rope, select, symm, tp_fused, zero1_comm  # noqa: F401


def extension_available() -> bool:
    return _ext.ext() is not None
