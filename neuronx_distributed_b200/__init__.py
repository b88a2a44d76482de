"""neuronx_distributed_b200 — an H100 (sm_90a) tensor/pipeline-parallel training and inference
library with the capabilities and public API of aws-neuron/neuronx-distributed.

Top-level exports mirror reference ``src/neuronx_distributed/__init__.py:1-19``.
"""
import os as _os

# NXD_EXPERIMENTAL=1 switches on every opt-in path that has not been timed on hardware yet (README.md, "Opt-in paths"): one
# flag to validate them together.  Individual flags set by the user win.  NXD_GEMM_MX / NXD_GEMM_F4 are not among them:
# NXD_GEMM_MX also quantises the activations (W8A8-MX numerics), a choice of the user's, and H100 has no FP4 tensor-core MMA.
_EXPERIMENTAL_FLAGS = ("NXD_FUSED_LMHEAD_CE", "NXD_MOE_TKG_KERNEL", "NXD_EMBEDDING_RS", "NXD_NVLS_A2A", "NXD_CP_PULL",
                       "NXD_GEMV_MX")
if _os.environ.get("NXD_EXPERIMENTAL", "0") == "1":
    for _f in _EXPERIMENTAL_FLAGS:
        _os.environ.setdefault(_f, "1")

from . import utils  # noqa: F401,E402
from . import ops  # noqa: F401,E402
from . import parallel_layers  # noqa: F401,E402
from .trainer.trainer import (  # noqa: F401,E402
    initialize_parallel_model,
    initialize_parallel_optimizer,
    neuronx_distributed_config,
)

from ._version import __version__  # noqa: E402,F401


def __getattr__(name):
    # heavier sub-systems are imported lazily so `import neuronx_distributed_b200` stays cheap
    import importlib

    lazy = {
        "pipeline": ".pipeline", "kernels": ".kernels", "trace": ".trace", "inference": ".inference",
        "modules": ".modules", "models": ".models", "optimizer": ".optimizer", "trainer": ".trainer",
        "quantization": ".quantization", "operators": ".operators", "lightning": ".lightning",
    }
    if name in lazy:
        return importlib.import_module(lazy[name], __name__)
    ckpt = {"save_checkpoint", "load_checkpoint", "has_checkpoint", "finalize_checkpoint", "CheckpointIOState"}
    if name in ckpt:
        mod = importlib.import_module(".trainer.checkpoint", __name__)
        return getattr(mod, name)
    # reference __init__.py:14-19: the v2 builder, the functional shard_checkpoint, the runtime model classes
    inf = {"ModelBuilder": ".trace.model_builder_v2", "shard_checkpoint": ".trace.functions", "NxDModel": ".trace.nxd_model",
           "BaseNxDModel": ".trace.nxd_model", "TorchScriptNxDModel": ".trace.nxd_model",
           "convert_nxd_model_to_torchscript_model": ".trace.nxd_model", "NxDParallelState": ".trace.parallel_context"}
    if name in inf:
        return getattr(importlib.import_module(inf[name], __name__), name)
    raise AttributeError(name)
