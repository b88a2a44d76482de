"""H100-specific inference pieces: launch plans (portable artefact / program IR), KV cache, bucketing, GQA sharding strategies,
HF adapter, benchmark helpers, checkpoint sharding.  The builder / functional units / runtime model are in ``trace/``."""
from .sharding import shard_state_dict_for_rank  # noqa: F401


def __getattr__(name):
    import importlib

    table = {
        # the builder / runtime classes live under ``trace/`` (the reference's module names); these are the v1 names
        "ModelBuilder": "..trace.model_builder", "NxDModel": "..trace.nxd_model", "BaseNxDModel": "..trace.nxd_model",
        "shard_checkpoint": "..trace.model_builder", "NxDParallelState": "..trace.parallel_context",
        "parallel_model_trace": "..trace.trace", "parallel_model_save": "..trace.trace", "parallel_model_load": "..trace.trace",
    }
    if name in table:
        return getattr(importlib.import_module(table[name], __name__), name)
    raise AttributeError(name)
