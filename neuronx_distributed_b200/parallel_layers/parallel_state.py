"""Process-group registry and rank topology.

Capability parity with reference ``src/neuronx_distributed/parallel_layers/parallel_state.py``
(``initialize_model_parallel`` :391-747, getters :833-1223, kv/token-shuffle/draft groups
:1285-1564, ``get_zero1_sharding_groups`` :1684-1706, ``rmsg`` :1648).

Design (H100-first, not a port):

* The rank grid is the same ``[PP, DP, CP, TP]`` / ``[PP, DP_exp, EP, TP]`` row-major layout
  (TP fastest varying) because checkpoint file names and ZeRO-1 shard ownership are defined
  by it.  It lives in an immutable :class:`RankMesh` that is pure python/numpy and can be
  built without any process group (``mesh_only=True``; what the unit tests use).
* NVSwitch gives uniform all-to-all bandwidth, so every Trainium topology special case in the
  reference (TP=4 non-contiguous groups, "ascending-descending ring", replica-group
  compression, logical-NeuronCore sizes) is dropped; ``lnc_size`` is accepted and ignored.
* Process groups are plain ``torch.distributed`` groups: NCCL on GPUs, gloo in CPU mode.  A
  separate gloo "control" group is kept for host metadata (pipeline shape exchange,
  symmetric-memory handle exchange) so control traffic never touches a CUDA stream.
* All state sits in one ``_STATE`` object instead of ~40 module globals.
"""
from __future__ import annotations

import enum
import os
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import torch.distributed as dist

from ..utils import cpu_mode, default_backend
from ..utils.logger import get_logger

logger = get_logger()

ProcessGroup = Any
GroupOrMesh = Union[ProcessGroup, List[List[int]]]


# --------------------------------------------------------------------------------------
# Pure topology
# --------------------------------------------------------------------------------------
@dataclass(frozen=True)
class RankMesh:
    """Pure description of which ranks form which parallel group."""

    world_size: int
    tp: int
    pp: int
    cp: int
    ep: int

    def __post_init__(self):
        if self.world_size % (self.tp * self.pp * self.cp) != 0:
            raise RuntimeError(
                f"invalid implied data parallel degree: world_size ({self.world_size}) is not divisible by "
                f"tensor_model_parallel_size ({self.tp}) x pipeline_model_parallel_size ({self.pp}) x "
                f"context_parallel_size ({self.cp})"
            )
        if self.world_size % (self.tp * self.pp * self.ep) != 0:
            raise RuntimeError(
                f"invalid implied expert data parallel degree: world_size ({self.world_size}) is not divisible by "
                f"tensor_model_parallel_size ({self.tp}) x pipeline_model_parallel_size ({self.pp}) x "
                f"expert_model_parallel_size ({self.ep})"
            )

    # degrees ------------------------------------------------------------------
    @property
    def dp(self) -> int:
        return self.world_size // (self.tp * self.pp * self.cp)

    @property
    def dp_exp(self) -> int:
        return self.world_size // (self.tp * self.pp * self.ep)

    # grids --------------------------------------------------------------------
    @property
    def grid(self) -> np.ndarray:
        return np.arange(self.world_size).reshape(self.pp, self.dp, self.cp, self.tp)

    @property
    def grid_exp(self) -> np.ndarray:
        return np.arange(self.world_size).reshape(self.pp, self.dp_exp, self.ep, self.tp)

    @staticmethod
    def _along(grid: np.ndarray, axis: int) -> List[List[int]]:
        moved = np.moveaxis(grid, axis, -1)
        return moved.reshape(-1, grid.shape[axis]).tolist()

    def tp_groups(self) -> List[List[int]]:
        return self._along(self.grid, 3)

    def dp_groups(self) -> List[List[int]]:
        return self._along(self.grid, 1)

    def pp_groups(self) -> List[List[int]]:
        return self._along(self.grid, 0)

    def cp_groups(self) -> List[List[int]]:
        return self._along(self.grid, 2)

    def ep_model_groups(self) -> List[List[int]]:
        return self._along(self.grid_exp, 2)

    def ep_data_groups(self) -> List[List[int]]:
        return self._along(self.grid_exp, 1)

    def coords(self, rank: int) -> Tuple[int, int, int, int]:
        """(pp, dp, cp, tp) coordinates of a global rank."""
        pp, dp, cp, tp = np.unravel_index(rank, self.grid.shape)
        return int(pp), int(dp), int(cp), int(tp)

    def coords_exp(self, rank: int) -> Tuple[int, int, int, int]:
        pp, dpe, ep, tp = np.unravel_index(rank, self.grid_exp.shape)
        return int(pp), int(dpe), int(ep), int(tp)

    def zero1_sharding_groups(self) -> List[List[int]]:
        """DP x CP merged groups over which ZeRO-1 shards optimizer state
        (reference parallel_state.py:1684-1706)."""
        g = self.grid  # [pp, dp, cp, tp]
        out = []
        for p in range(self.pp):
            for t in range(self.tp):
                out.append(g[p, :, :, t].reshape(-1).tolist())
        return out

    def cp_ring_pairs(self, rank: int) -> List[Tuple[int, int]]:
        """(src, tgt) pairs of the ring this rank's CP group uses for ring attention
        (reference parallel_state.py:737-742)."""
        for grp in self.cp_groups():
            if rank in grp:
                n = len(grp)
                return [(grp[i], grp[(i + 1) % n]) for i in range(n)]
        return []


ParallelGroups = RankMesh  # name kept for API familiarity (reference :105)


def ascending_ring_PG_group(lnc_size: int = 1, cluster_ranks_nonexp=None, cluster_ranks_exp=None, tp: int = 1, dp: int = 1,
                            pp: int = 1, ep_model_degree: int = 1, ep_data_degree: int = 1, cp: int = 1) -> RankMesh:
    """Rank-placement policy: consecutive ranks form a TP group (reference parallel_state.py:107-175).

    Behind an NVSwitch every GPU is one hop from every other, so this is the ONLY placement policy here: it keeps a TP
    group inside one NVLink domain (8 GPUs) and puts DP / PP across nodes.  The reference's second policy
    (:177-325, interleaved rings for the Trn2 torus) has no H100 counterpart and maps to this one.
    """
    return RankMesh(tp * dp * pp * cp, tp, pp, cp, ep_model_degree)


ascending_descending_ring_PG_group = ascending_ring_PG_group


class PG_Group_Logic(enum.Enum):  # noqa: N801  (reference spelling, :326-335)
    """Callable enum of rank-placement policies; both members resolve to the NVSwitch placement."""

    LOGIC1 = ("ascending", "Ascending Ring PG Group")
    LOGIC2 = ("ascending_descending", "Ascending Descending Ring PG Group")

    def __init__(self, ident: str, description: str):
        self.ident, self.description = ident, description

    @property
    def func(self):
        return ascending_ring_PG_group

    def __call__(self, *args, **kwargs):
        return ascending_ring_PG_group(*args, **kwargs)


def get_logic_chosen(lnc_size: int = 1, hardware_type: Any = None, tp: int = 1):
    """Reference parallel_state.py:341-357 picks a placement by hardware generation; H100 has one."""
    return PG_Group_Logic.LOGIC1


def arrange_kv_groups(
    num_tensor_model_parallel_groups: int = 1,
    tensor_model_parallel_size: int = 1,
    kv_shared_group_size: int = 1,
    sequential_ranks_in_group: bool = False,
    hardware_type: Any = None,
    adjacent_replication: bool = False,
) -> List[List[int]]:
    """Ranks that hold replicas of the same KV head (GQA with kv_heads < tp).

    ``sequential_ranks_in_group``/``adjacent_replication`` → [[0,1],[2,3]]; default is the
    interleaved layout [[0,2],[1,3]] (reference parallel_state.py:1605-1645).  The reference
    picks the adjacent layout by hardware generation; ``hardware_type="trn2"`` is accepted
    and means ``adjacent_replication=True``, anything else leaves the flags in charge.
    """
    if isinstance(hardware_type, str) and hardware_type.lower() == "trn2":
        adjacent_replication = True
    tp, k = tensor_model_parallel_size, kv_shared_group_size
    groups: List[List[int]] = []
    if sequential_ranks_in_group or adjacent_replication:
        total = num_tensor_model_parallel_groups * tp
        return [list(range(i, i + k)) for i in range(0, total, k)]
    step = tp // k
    for i in range(num_tensor_model_parallel_groups):
        for j in range(step):
            groups.append(list(range(i * tp + j, (i + 1) * tp, step)))
    return groups


# --------------------------------------------------------------------------------------
# Registry
# --------------------------------------------------------------------------------------
@dataclass
class _Group:
    mesh: List[List[int]]
    pg: Optional[ProcessGroup] = None

    def my_ranks(self, rank: int) -> List[int]:
        for g in self.mesh:
            if rank in g:
                return g
        raise AssertionError(f"rank {rank} not in any group of {self.mesh}")


@dataclass
class _State:
    mesh: Optional[RankMesh] = None
    rank: int = 0
    groups: Dict[str, _Group] = field(default_factory=dict)
    overrides: Dict[str, int] = field(default_factory=dict)
    kv_group_size: Optional[int] = None
    token_shuffle_group_size: Optional[int] = None
    draft_group_size: Optional[int] = None
    control_pg: Optional[ProcessGroup] = None
    pp_gloo_pg: Optional[ProcessGroup] = None
    aot_mode: bool = False
    shared_weight_pgs: Dict[Tuple[int, ...], ProcessGroup] = field(default_factory=dict)


_STATE = _State()


def _new_group_family(mesh: List[List[int]], backend: Optional[str] = None) -> Optional[ProcessGroup]:
    """Collectively create one process group per entry of ``mesh``; return mine.

    Every rank must call ``new_group`` for every entry, in the same order."""
    rank = dist.get_rank()
    mine = None
    for ranks in mesh:
        pg = dist.new_group(ranks=ranks, backend=backend or default_backend())
        if rank in ranks:
            mine = pg
    return mine


def _register(name: str, mesh: List[List[int]], build_pg: bool = True, backend: Optional[str] = None) -> None:
    pg = _new_group_family(mesh, backend) if build_pg else None
    _STATE.groups[name] = _Group(mesh=mesh, pg=pg)


def initialize_model_parallel(
    tensor_model_parallel_size: int = 1,
    pipeline_model_parallel_size: int = 1,
    expert_model_parallel_size: int = 1,
    skip_collective_init: bool = False,
    lnc_size: int = 1,
    mesh_only: bool = False,
    context_parallel_size: int = 1,
    world_size: Optional[int] = None,
    rank: Optional[int] = None,
) -> Optional[RankMesh]:
    """Build every parallel group for this job.

    ``mesh_only=True`` returns the :class:`RankMesh` without touching ``torch.distributed``
    (pass ``world_size``).  ``lnc_size`` and ``skip_collective_init`` are accepted for
    source compatibility; NCCL needs no collective bring-up graph.
    """
    del lnc_size
    if mesh_only:
        assert world_size is not None or dist.is_initialized()
        ws = world_size if world_size is not None else dist.get_world_size()
        return RankMesh(
            ws,
            min(tensor_model_parallel_size, ws),
            min(pipeline_model_parallel_size, ws),
            min(context_parallel_size, ws),
            min(expert_model_parallel_size, ws),
        )

    assert dist.is_initialized(), "torch.distributed must be initialised before initialize_model_parallel"
    if model_parallel_is_initialized():
        raise RuntimeError("model parallel state is already initialized; call destroy_model_parallel() first")
    ws = dist.get_world_size()
    me = dist.get_rank()
    mesh = RankMesh(
        ws,
        min(tensor_model_parallel_size, ws),
        min(pipeline_model_parallel_size, ws),
        min(context_parallel_size, ws),
        min(expert_model_parallel_size, ws),
    )
    logger.info(
        "> initializing model parallel: tp=%d pp=%d cp=%d dp=%d ep=%d dp_exp=%d world=%d",
        mesh.tp, mesh.pp, mesh.cp, mesh.dp, mesh.ep, mesh.dp_exp, ws,
    )
    _STATE.mesh = mesh
    _STATE.rank = me

    _STATE.groups["world"] = _Group(mesh=[list(range(ws))], pg=dist.group.WORLD)
    _register("tp", mesh.tp_groups())
    _register("dp", mesh.dp_groups())
    _register("pp", mesh.pp_groups())
    _register("exp_dp", mesh.ep_data_groups())
    _register("ep", mesh.ep_model_groups())
    _register("cp", mesh.cp_groups())
    # ZeRO-1 shards across DP x CP
    if mesh.cp > 1:
        _register("zero1", mesh.zero1_sharding_groups())
    else:
        _STATE.groups["zero1"] = _STATE.groups["dp"]
    # Host-side control plane (gloo) — metadata, handle exchange.  In CPU mode the world
    # group already is gloo.
    if cpu_mode():
        _STATE.control_pg = dist.group.WORLD
    else:
        _STATE.control_pg = dist.new_group(ranks=list(range(ws)), backend="gloo")

    if not skip_collective_init and not cpu_mode():
        # one tiny all-reduce so NCCL communicators for WORLD come up before the first
        # timed step (reference does the same with a dummy graph, :647-657)
        t = torch.zeros(1, device=torch.device("cuda", torch.cuda.current_device()))
        dist.all_reduce(t)
    return mesh


def model_parallel_is_initialized() -> bool:
    return _STATE.mesh is not None


def destroy_model_parallel() -> None:
    """Forget all groups (reference :1226-1283).  Process groups other than WORLD are
    destroyed so tests can re-initialise with a different layout."""
    global _STATE
    seen = set()
    for name, g in list(_STATE.groups.items()):
        if name == "world" or g.pg is None or id(g.pg) in seen:
            continue
        seen.add(id(g.pg))
        try:
            if g.pg is not dist.group.WORLD:
                dist.destroy_process_group(g.pg)
        except Exception:  # pragma: no cover - best effort
            pass
    for pg in [_STATE.control_pg, _STATE.pp_gloo_pg, *_STATE.shared_weight_pgs.values()]:
        if pg is not None and pg is not dist.group.WORLD and id(pg) not in seen:
            seen.add(id(pg))
            try:
                dist.destroy_process_group(pg)
            except Exception:  # pragma: no cover
                pass
    _STATE = _State()
    try:
        from .. import ops

        ops.symm.reset()
    except Exception:
        pass


def _need() -> RankMesh:
    assert _STATE.mesh is not None, "model parallel state is not initialized"
    return _STATE.mesh


def get_mesh() -> RankMesh:
    return _need()


def _group(name: str, as_list: bool) -> GroupOrMesh:
    _need()
    g = _STATE.groups.get(name)
    assert g is not None, f"{name} group is not initialized"
    return g.mesh if as_list else g.pg


def group_name(pg: ProcessGroup) -> Optional[str]:
    """Registry name of a process group ("tp", "dp", "world", …) or ``None`` — used to store groups symbolically (launch plans)."""
    for name, g in _STATE.groups.items():
        if g.pg is pg:
            return name
    if pg is None or (dist.is_initialized() and pg is dist.group.WORLD):
        return "__default__"
    return None


def group_by_name(name: str) -> Optional[ProcessGroup]:
    if name == "__default__":
        return dist.group.WORLD
    g = _STATE.groups.get(name)
    assert g is not None, f"process group {name!r} is not initialized"
    return g.pg


def _my_ranks(name: str) -> List[int]:
    return _STATE.groups[name].my_ranks(_STATE.rank)


# ---- world -------------------------------------------------------------------------
def get_world_group(as_list: bool = False) -> GroupOrMesh:
    return _group("world", as_list)


def get_control_group() -> ProcessGroup:
    """gloo group spanning the world for host metadata."""
    _need()
    return _STATE.control_pg


def is_global_rank_zero() -> bool:
    return (dist.get_rank() if dist.is_initialized() else 0) == 0


# ---- tensor parallel ---------------------------------------------------------------
def get_tensor_model_parallel_group(as_list: bool = False) -> GroupOrMesh:
    return _group("tp", as_list)


def get_tensor_model_parallel_replica_groups() -> List[List[int]]:
    return _group("tp", True)


def _set_override(key: str, value) -> None:
    """Manual override of a size / rank (offline tools that play every rank in one process); ``None`` removes it."""
    if value is None:
        _STATE.overrides.pop(key, None)
    else:
        _STATE.overrides[key] = value


def get_tensor_model_parallel_size() -> int:
    if "tp_size" in _STATE.overrides:
        return _STATE.overrides["tp_size"]
    return _need().tp


def set_tensor_model_parallel_size(world_size: int) -> None:
    _set_override("tp_size", world_size)


def get_tensor_model_parallel_rank() -> int:
    if "tp_rank" in _STATE.overrides:
        return _STATE.overrides["tp_rank"]
    return _need().coords(_STATE.rank)[3]


def set_tensor_model_parallel_rank(rank: int) -> None:
    _set_override("tp_rank", rank)


def get_tensor_model_parallel_src_rank() -> int:
    """Global rank of tp-rank 0 in my TP group."""
    return _my_ranks("tp")[0]


def get_tensor_model_parallel_ranks() -> List[int]:
    return _my_ranks("tp")


# ---- data parallel -----------------------------------------------------------------
def get_data_parallel_group(as_list: bool = False) -> GroupOrMesh:
    return _group("dp", as_list)


def get_data_parallel_replica_groups() -> List[List[int]]:
    return _group("dp", True)


def get_data_parallel_size() -> int:
    return _need().dp


def get_data_parallel_rank() -> int:
    return _need().coords(_STATE.rank)[1]


def get_data_parallel_src_rank() -> int:
    return _my_ranks("dp")[0]


def get_data_parallel_ranks() -> List[int]:
    return _my_ranks("dp")


# ---- expert parallel ---------------------------------------------------------------
def get_expert_model_parallel_group(as_list: bool = False) -> GroupOrMesh:
    return _group("ep", as_list)


def get_expert_model_parallel_replica_groups() -> List[List[int]]:
    return _group("ep", True)


def get_expert_model_parallel_size() -> int:
    if "ep_size" in _STATE.overrides:
        return _STATE.overrides["ep_size"]
    return _need().ep


def set_expert_model_parallel_size(world_size: int) -> None:
    _set_override("ep_size", world_size)


def get_expert_model_parallel_rank() -> int:
    if "ep_rank" in _STATE.overrides:
        return _STATE.overrides["ep_rank"]
    return _need().coords_exp(_STATE.rank)[2]


def set_expert_model_parallel_rank(rank: int) -> None:
    _set_override("ep_rank", rank)


def get_expert_data_parallel_group(as_list: bool = False) -> GroupOrMesh:
    return _group("exp_dp", as_list)


def get_expert_data_parallel_replica_groups() -> List[List[int]]:
    return _group("exp_dp", True)


def get_expert_data_parallel_size() -> int:
    return _need().dp_exp


def get_expert_data_parallel_rank() -> int:
    return _need().coords_exp(_STATE.rank)[1]


def get_expert_parallel_rank_from_global_rank(rank: int, expert_parallel_group: Any = None) -> int:
    return _need().coords_exp(rank)[2]


def get_experts_for_expert_parallel_rank(
    expert_parallel_rank: int,
    total_number_of_experts: int,
    expert_model_parallel_size: int,
    expert_distribution: Optional[List[List[int]]] = None,
) -> List[int]:
    """Indices of the experts an EP rank owns: contiguous blocks unless an explicit
    distribution is given (reference :999-1027)."""
    if expert_distribution is not None:
        return list(expert_distribution[expert_parallel_rank])
    assert total_number_of_experts % expert_model_parallel_size == 0
    per = total_number_of_experts // expert_model_parallel_size
    return list(range(expert_parallel_rank * per, (expert_parallel_rank + 1) * per))


# ---- pipeline parallel -------------------------------------------------------------
def get_pipeline_model_parallel_group(as_list: bool = False) -> GroupOrMesh:
    return _group("pp", as_list)


def get_pipeline_model_parallel_replica_groups() -> List[List[int]]:
    return _group("pp", True)


def get_pipeline_model_parallel_size() -> int:
    return _need().pp


def get_pipeline_model_parallel_rank() -> int:
    return _need().coords(_STATE.rank)[0]


def get_pipeline_model_parallel_ranks() -> List[int]:
    return _my_ranks("pp")


def get_pipeline_model_parallel_next_rank() -> int:
    ranks = _my_ranks("pp")
    return ranks[(get_pipeline_model_parallel_rank() + 1) % len(ranks)]


def get_pipeline_model_parallel_prev_rank() -> int:
    ranks = _my_ranks("pp")
    return ranks[(get_pipeline_model_parallel_rank() - 1) % len(ranks)]


def get_pipeline_model_parallel_sr_group(parity: Optional[bool] = None) -> List[List[int]]:
    """2-rank (sender, receiver) pairs along every PP group, optionally only those whose
    sender has even/odd pp-rank (reference :1119-1137).  NCCL has native send/recv so the
    engine does not need process groups for these; kept as topology information."""
    pairs: List[List[int]] = []
    for ranks in _group("pp", True):
        for i in range(len(ranks) - 1):
            if parity is None or bool(i % 2) == parity:
                pairs.append([ranks[i], ranks[i + 1]])
    return pairs


def get_next_rank_group(as_list: bool = False) -> GroupOrMesh:
    if as_list:
        return [[_STATE.rank, get_pipeline_model_parallel_next_rank()]]
    return _group("pp", False)


def get_prev_rank_group(as_list: bool = False) -> GroupOrMesh:
    if as_list:
        return [[get_pipeline_model_parallel_prev_rank(), _STATE.rank]]
    return _group("pp", False)


get_next_rank_replica_groups = lambda: get_next_rank_group(True)  # noqa: E731
get_prev_rank_replica_groups = lambda: get_prev_rank_group(True)  # noqa: E731


def initialize_pp_gloo_groups() -> None:
    """gloo groups mirroring the PP groups, for python-object metadata exchange
    (reference :1387-1409)."""
    if _STATE.pp_gloo_pg is not None:
        return
    if cpu_mode():
        _STATE.pp_gloo_pg = _group("pp", False)
    else:
        _STATE.pp_gloo_pg = _new_group_family(_group("pp", True), backend="gloo")


def get_pp_gloo_group() -> ProcessGroup:
    if _STATE.pp_gloo_pg is None:
        initialize_pp_gloo_groups()
    return _STATE.pp_gloo_pg


def is_tcp_store_available() -> bool:
    try:
        return dist.distributed_c10d._get_default_store() is not None
    except Exception:
        return False


def get_tcp_store():
    return dist.distributed_c10d._get_default_store()


# ---- context parallel --------------------------------------------------------------
def get_context_model_parallel_group(as_list: bool = False) -> GroupOrMesh:
    return _group("cp", as_list)


def get_context_model_parallel_replica_groups() -> List[List[int]]:
    return _group("cp", True)


def get_context_model_parallel_size() -> int:
    if "cp_size" in _STATE.overrides:
        return _STATE.overrides["cp_size"]
    return _need().cp


def set_context_model_parallel_size(world_size: int) -> None:
    _set_override("cp_size", world_size)


def get_context_model_parallel_rank() -> int:
    return _need().coords(_STATE.rank)[2]


def get_context_model_parallel_ranks() -> List[int]:
    return _my_ranks("cp")


def get_context_model_parallel_src_tgt_pairs() -> List[Tuple[int, int]]:
    return _need().cp_ring_pairs(_STATE.rank)


# ---- ZeRO-1 ------------------------------------------------------------------------
def get_zero1_sharding_groups() -> List[List[int]]:
    return _need().zero1_sharding_groups()


def get_zero1_sharding_group() -> ProcessGroup:
    return _group("zero1", False)


def get_zero1_sharding_ranks() -> List[int]:
    return _my_ranks("zero1")


# ---- auxiliary groups --------------------------------------------------------------
def initialize_kv_group(kv_shared_group_size: int = 1, sequential_ranks_in_group: bool = False) -> None:
    """Groups of TP ranks holding replicas of the same KV head (reference :1473-1501)."""
    if "kv" in _STATE.groups:
        assert kv_shared_group_size == _STATE.kv_group_size, "only one KV replication factor is supported"
        return
    m = _need()
    assert m.tp % kv_shared_group_size == 0
    _STATE.kv_group_size = kv_shared_group_size
    mesh = arrange_kv_groups(m.world_size // m.tp, m.tp, kv_shared_group_size, sequential_ranks_in_group)
    _register("kv", mesh)


def get_kv_shared_group(as_list: bool = False) -> GroupOrMesh:
    return _group("kv", as_list)


def get_kv_shared_replica_groups() -> List[List[int]]:
    return _group("kv", True)


def get_kv_shared_group_size() -> int:
    assert _STATE.kv_group_size is not None, "kv group is not initialized"
    return _STATE.kv_group_size


def destroy_kv_group() -> None:
    g = _STATE.groups.pop("kv", None)
    _STATE.kv_group_size = None
    if g is not None and g.pg is not None:
        dist.destroy_process_group(g.pg)


def initialize_token_shuffle_group(token_shuffle_group_size: int = 1) -> None:
    """Sub-groups of the DP group used by MoE token shuffling (reference :1285-1343)."""
    if "token_shuffle" in _STATE.groups:
        assert token_shuffle_group_size == _STATE.token_shuffle_group_size
        return
    m = _need()
    assert token_shuffle_group_size <= m.dp and m.dp % token_shuffle_group_size == 0
    _STATE.token_shuffle_group_size = token_shuffle_group_size
    grid = np.arange(m.world_size).reshape(m.pp, m.dp // token_shuffle_group_size, token_shuffle_group_size, m.tp)
    _register("token_shuffle", RankMesh._along(grid, 2))


def get_token_shuffle_group(as_list: bool = False) -> GroupOrMesh:
    return _group("token_shuffle", as_list)


def get_token_shuffle_replica_groups() -> List[List[int]]:
    return _group("token_shuffle", True)


def get_token_shuffle_group_size() -> int:
    assert _STATE.token_shuffle_group_size is not None
    return _STATE.token_shuffle_group_size


def destroy_token_shuffle_group() -> None:
    g = _STATE.groups.pop("token_shuffle", None)
    _STATE.token_shuffle_group_size = None
    if g is not None and g.pg is not None:
        dist.destroy_process_group(g.pg)


def initialize_speculative_draft_group(group_size: int = 1) -> None:
    """Consecutive-rank sub-groups of TP used by a smaller draft model (reference :1533-1564)."""
    if "draft" in _STATE.groups:
        assert group_size == _STATE.draft_group_size
        return
    m = _need()
    assert m.tp % group_size == 0
    _STATE.draft_group_size = group_size
    _register("draft", [list(range(i, i + group_size)) for i in range(0, m.world_size, group_size)])


def get_speculative_draft_group(as_list: bool = False) -> GroupOrMesh:
    return _group("draft", as_list)


def get_speculative_draft_replica_groups() -> List[List[int]]:
    return _group("draft", True)


def create_pg_with_ranks(ranks: Sequence[int]) -> ProcessGroup:
    """Collective creation of a group for ``ranks`` — every rank in the *world* must call this
    with the same sequence of rank lists (used for tied weights across PP stages; reference
    :1421-1470).  Groups are cached by rank tuple."""
    key = tuple(ranks)
    if key not in _STATE.shared_weight_pgs:
        _STATE.shared_weight_pgs[key] = dist.new_group(ranks=list(ranks), backend=default_backend())
    return _STATE.shared_weight_pgs[key]


def gather_python_object(obj: Any, group: ProcessGroup) -> List[Any]:
    out: List[Any] = [None] * dist.get_world_size(group)
    dist.all_gather_object(out, obj, group=group)
    return out


def set_aot_mode(mode: bool) -> None:
    _STATE.aot_mode = mode


def get_aot_mode() -> bool:
    return _STATE.aot_mode


# ---- messages ----------------------------------------------------------------------
def rmsg(msg: str) -> str:
    """Prefix a message with this rank's parallel coordinates (reference :1648-1667)."""
    if model_parallel_is_initialized():
        pp, dp, cp, tp = _need().coords(_STATE.rank)
    else:
        pp = dp = cp = tp = -1
    g = dist.get_rank() if dist.is_initialized() else int(os.environ.get("RANK", 0))
    return f"[rank_{g}_pp{pp}_tp{tp}_dp{dp}_cp{cp}] {msg}"


def rmsg_ep(msg: str) -> str:
    return (
        f"[pp{get_pipeline_model_parallel_rank()}|ep{get_expert_model_parallel_rank()}|"
        f"tp{get_tensor_model_parallel_rank()}|dp{get_data_parallel_rank()}] {msg}"
    )


def get_rank_info_str() -> str:
    if model_parallel_is_initialized():
        return (
            f"DP_{get_data_parallel_rank()}_TP_{get_tensor_model_parallel_rank()}"
            f"_PP_{get_pipeline_model_parallel_rank()}"
        )
    return "model_parallel_uninitialized"


def initialize_fallback_parallel_state() -> None:
    """Single-process world so TP layers can be constructed in plain scripts
    (reference parallel_layers/utils.py:318-335)."""
    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29521")
        dist.init_process_group(default_backend(), rank=0, world_size=1)
    if not model_parallel_is_initialized():
        initialize_model_parallel(1, 1, 1)
