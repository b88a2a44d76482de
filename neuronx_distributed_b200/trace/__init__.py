"""``neuronx_distributed.trace`` import paths (reference ``trace/__init__.py``).  "Tracing / compiling" a
bucket means validating its signature and capturing it into a CUDA graph; the builder, the functional units and the runtime model
live here under the reference's module names, the H100-specific pieces (launch plans, KV cache, bucketing, GQA sharding, HF
adapter) in :mod:`neuronx_distributed_b200.inference`."""
from .model_builder import ModelBuilder  # noqa: F401
from ..inference.sharding import shard_state_dict_for_rank  # noqa: F401
from .trace import parallel_model_load, parallel_model_save, parallel_model_trace  # noqa: F401
from .spmd import NxDModel, SPMDBucketModelScript  # noqa: F401


def __getattr__(name):
    import importlib

    inf = importlib.import_module("..inference", __name__)
    return getattr(inf, name)
