"""Routed expert MLPs — dispatch over execution modes (reference ``modules/moe/expert_mlps_v2.py:1407-1500``):

* **all-experts**: every local expert processes every token, results masked/weighted — best for tiny token counts
  (decode) where the weights, not the activations, dominate memory traffic;
* **capacity-factor**: each expert takes at most ``C = ceil(cf·T·k/E)`` tokens in routing order, the rest are
  dropped (position-in-expert via cumsum, reference :484-593); batched ``[E, C, H]`` GEMMs;
* **blockwise (dropless)**: :mod:`.blockwise`;
* **selective loading** (decode / short speculation windows): only the ``T·k`` chosen experts' weights are touched;
* **expert parallel** (training): capacity-factor layout + all-to-all dispatch/combine over the EP group
  (``enter/exit_expert_parallel_region``, reference experts.py:174-214); inference masks to local experts instead.

Mode selection follows the reference's ``forward`` (:1407-1500) with one deliberate difference: a ``capacity_factor`` of
``None`` ("full capacity") in training runs the dropless blockwise path once ``T·k`` reaches a block instead of pushing
every token through every expert — same result, 1/E·k of the FLOPs (the grouped wgmma GEMM makes dropless the cheap
option here).
"""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import nn

from ...parallel_layers import mappings
from ...parallel_layers import parallel_state as ps
from ...parallel_layers.layers import ProcessGroupSafeDeepcopy
from ...utils.logger import get_logger
from .blockwise import blockwise_expert_mlp, build_block_metadata
from .experts import Experts
from .model_utils import ACT2FN, DEFAULT_SELECTIVE_LOADING_THRESHOLD, create_spmd_ranks as _create_spmd_ranks
from .moe_configs import BlockwiseMatmulConfig, RoutedExpertsMLPOpsConfig

logger = get_logger()


class ExpertMLPsV2(ProcessGroupSafeDeepcopy, nn.Module):
    def __init__(self, routed_experts_mlp_config: RoutedExpertsMLPOpsConfig,
                 blockwise_matmul_config: Optional[BlockwiseMatmulConfig] = None, sequence_parallel_enabled: bool = False,
                 dtype: torch.dtype = torch.float32, device=None, tensor_model_parallel_group=None,
                 expert_model_parallel_group=None, is_prefill: bool = True, return_bias: bool = False,
                 init_method=None, output_layer_init_method=None, enabled_hybrid_sharding: bool = False,
                 cte_tensor_model_parallel_group=None, cte_expert_model_parallel_group=None,
                 tkg_tensor_model_parallel_group=None, tkg_expert_model_parallel_group=None):
        super().__init__()
        c = routed_experts_mlp_config
        self.validate_routed_experts_configs(c)
        self.routed_experts_mlp_config = self.cfg = c
        self.blockwise_matmul_config = self.bw = blockwise_matmul_config or BlockwiseMatmulConfig.default()
        self.num_experts, self.top_k = c.num_experts, c.top_k
        self.sequence_parallel_enabled, self.is_prefill, self.return_bias = sequence_parallel_enabled, is_prefill, return_bias
        self.dtype, self.device = dtype, device
        self.enabled_hybrid_sharding = enabled_hybrid_sharding
        self.tensor_parallel_group = tensor_model_parallel_group
        if c.input_layer_init_method is None and init_method is not None:
            c.input_layer_init_method = init_method
        if c.output_layer_init_method is None and output_layer_init_method is not None:
            c.output_layer_init_method = output_layer_init_method
        if ps.model_parallel_is_initialized():
            self.ep = ps.get_expert_model_parallel_size() if expert_model_parallel_group is None else \
                torch.distributed.get_world_size(expert_model_parallel_group)
        else:
            self.ep = 1
        if enabled_hybrid_sharding:
            # prefill and decode shard the same experts over different (tp, ep) factorizations of the same ranks
            # (reference :148-177): two weight sets, filled from one checkpoint by the preshard hook
            self.mlp_op = self._build_experts(cte_tensor_model_parallel_group, cte_expert_model_parallel_group, True)
            self.mlp_op_tkg = self._build_experts(tkg_tensor_model_parallel_group, tkg_expert_model_parallel_group, False)
        else:
            self.mlp_op = self._build_experts(tensor_model_parallel_group, expert_model_parallel_group, is_prefill)
        self.local_expert_ids = self.mlp_op.local_expert_ids
        self.spmd_rank = None
        if c.enable_spmd_rank:
            from ...parallel_layers.layers import SPMDRank

            world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
            self.spmd_rank = SPMDRank(world_size=world)

    @property
    def capacity_factor(self):
        return self.routed_experts_mlp_config.capacity_factor

    @capacity_factor.setter
    def capacity_factor(self, v):
        self.routed_experts_mlp_config.capacity_factor = v

    def _build_experts(self, tp_group, ep_group, is_prefill: bool) -> Experts:
        c = self.routed_experts_mlp_config
        return Experts(
            c.num_experts, c.hidden_size, c.intermediate_size, c.hidden_act, c.glu_mlp, c.glu_type, c.capacity_factor,
            reduce_output=False, dtype=self.dtype, device=self.device, input_layer_init_method=c.input_layer_init_method,
            output_layer_init_method=c.output_layer_init_method, tensor_model_parallel_group=tp_group,
            hidden_act_scaling_factor=c.hidden_act_scaling_factor, hidden_act_bias=c.hidden_act_bias,
            gate_clamp_upper_limit=c.gate_clamp_upper_limit, gate_clamp_lower_limit=c.gate_clamp_lower_limit,
            up_clamp_upper_limit=c.up_clamp_upper_limit, up_clamp_lower_limit=c.up_clamp_lower_limit, bias=c.bias,
            expert_model_parallel_group=ep_group, is_prefill=is_prefill)

    def get_mlp_op(self) -> Experts:
        if self.enabled_hybrid_sharding and not self.training and not self._decode_hint:
            return self.mlp_op
        if self.enabled_hybrid_sharding and self._decode_hint:
            return self.mlp_op_tkg
        return self.mlp_op

    _decode_hint = False

    def get_spmd_rank(self):
        return None if self.spmd_rank is None else self.spmd_rank.get_rank()

    def preshard_hook(self, model_state_dict, prefix: str) -> None:
        """Full-checkpoint fix-ups before sharding (reference :197-258): SPMD rank entry; hybrid sharding duplicates the
        expert weights under the decode copy's prefix so both factorizations are cut from the same tensors."""
        base = prefix[: prefix.index("mlp_op")] if "mlp_op" in prefix else (prefix[: prefix.rfind(".") + 1] if "." in prefix else "")
        if self.spmd_rank is not None:
            _create_spmd_ranks(model_state_dict, base, self.spmd_rank.world_size)
        if self.enabled_hybrid_sharding:
            duplicate_and_replace_prefixes(base + "mlp_op.", base + "mlp_op_tkg.", model_state_dict)

    # ------------------------------------------------------------------ helpers
    @staticmethod
    def validate_routed_experts_configs(routed_experts_mlp_config: RoutedExpertsMLPOpsConfig) -> None:
        c = routed_experts_mlp_config      # reference parameter names in the signature
        if not (0 < c.top_k <= c.num_experts):
            raise ValueError(f"Invalid top_k={c.top_k} for num_experts={c.num_experts}")
        if c.hidden_act not in ACT2FN:
            raise ValueError(f"Unknown activation: {c.hidden_act} ; Supported: {list(ACT2FN.keys())}")
        if c.capacity_factor is not None and c.capacity_factor >= c.num_experts / c.top_k:
            c.capacity_factor = None                       # cannot drop anything: full capacity

    @staticmethod
    def get_expert_mask(expert_index: torch.Tensor, num_experts: int) -> torch.Tensor:
        """``[T, k]`` indices → k-hot ``[T, E]`` mask (float64 so later masked products stay exact)."""
        return torch.zeros(expert_index.shape[0], num_experts, dtype=torch.float64, device=expert_index.device
                           ).scatter_add_(1, expert_index, torch.ones_like(expert_index, dtype=torch.float64))

    @staticmethod
    def get_expert_affinities_masked(expert_affinities: torch.Tensor, expert_mask: torch.Tensor,
                                     normalize_top_k_affinities: bool) -> torch.Tensor:
        a = expert_affinities.masked_fill(expert_mask == 0, 0)
        if normalize_top_k_affinities:
            a = a / a.abs().sum(-1, keepdim=True).clamp(min=1e-12)
        return a

    def mask_padding_tokens(self, expert_mask, expert_affinities_masked, padding_mask):
        """Zero the routing of padded tokens (``padding_mask [B, S]``: 1 = real token)."""
        if padding_mask is None:
            return expert_mask, expert_affinities_masked
        m = padding_mask.reshape(-1, 1)
        expert_affinities_masked = expert_affinities_masked * m.to(expert_affinities_masked.dtype)
        if expert_mask is not None:
            expert_mask = expert_mask * m.to(expert_mask.dtype)
        return expert_mask, expert_affinities_masked

    def get_sp_expert_masks_index(self, expert_affinities_masked: torch.Tensor, expert_index: torch.Tensor):
        """Router ran on the sequence shard: gather its outputs over the TP group (inference SP flow)."""
        a, i = (mappings.gather_from_sequence_parallel_region(t, 0, to_model_parallel=False,
                                                              process_group=self.tensor_parallel_group)
                for t in (expert_affinities_masked, expert_index))
        return a, (a > 0).to(torch.float64), i

    def get_full_expert_affinities_masked(self, expert_affinities: torch.Tensor, expert_index: torch.Tensor) -> torch.Tensor:
        a = self._topk_affinities(expert_affinities, expert_index)
        return mappings.gather_from_sequence_parallel_region(a, 0, to_model_parallel=False, process_group=self.tensor_parallel_group)

    def maybe_get_expert_affinities_masked(self, expert_index, expert_affinities, expert_affinities_masked_full=None,
                                           padding_mask=None):
        if expert_affinities_masked_full is not None:
            return expert_affinities_masked_full
        return self._topk_affinities(expert_affinities, expert_index)

    def _topk_affinities(self, aff: torch.Tensor, idx: torch.Tensor, padding_mask=None) -> torch.Tensor:
        """[T, E] affinities keeping only the chosen experts (optionally re-normalised over them)."""
        mask = torch.zeros_like(aff).scatter_(1, idx, 1.0)
        a = aff * mask
        if self.cfg.normalize_top_k_affinities:
            a = a / a.sum(-1, keepdim=True).clamp(min=1e-9)
        if padding_mask is not None:
            a = a * padding_mask.reshape(-1, 1).to(a.dtype)
        return a

    def get_blockwise_expert_and_token_mapping(self, total_tokens: int, num_blocks: int, expert_mask: torch.Tensor,
                                               expert_index: torch.Tensor, block_size: Optional[int] = None, **_unused):
        """``(block_to_expert [N], token_position_to_id [N·B])`` for the dropless layout (reference :1208-1348); computed
        on device by a sort + prefix sums (``blockwise.build_block_metadata``), padding slots are ``-1``."""
        b2e, tp2id, _ = build_block_metadata(expert_index, self.num_experts, block_size or self.bw.block_size)
        return b2e[:num_blocks], tp2id[: num_blocks * (block_size or self.bw.block_size)]

    # ------------------------------------------------------------------ redundant experts (reference :919-1077)
    # An ``expert_distribution`` may host a hot logical expert on several EP ranks (or twice on one).  Tokens routed to such
    # an expert are split by token position between its replicas so that nothing is computed twice.
    @staticmethod
    def allocate_token_blocks(local_redudancy_degree: torch.Tensor, tokens_per_expert):
        """``local_redudancy_degree [ep, E]`` (replicas of expert e hosted by EP rank g) → inclusive token-position ranges
        ``(start [ep, E], end [ep, E])``: expert e's ``tokens_per_expert`` positions are cut into equal blocks, one per
        replica, handed out in EP-rank order; the last replica also takes the remainder."""
        deg = local_redudancy_degree.to(torch.int32)
        total = deg.sum(0)                                                       # replicas per expert
        upto = torch.cumsum(deg, 0, dtype=torch.int32)
        before = upto - deg
        tpe = torch.as_tensor(tokens_per_expert, dtype=torch.int32, device=deg.device)
        block = (tpe // total.clamp(min=1)).to(torch.int32)
        rem = (tpe % total.clamp(min=1)).to(torch.int32)
        start = before * block
        end = upto * block - 1 + (upto == total).to(torch.int32) * rem
        return start.to(torch.int32), end.to(torch.int32)

    @staticmethod
    def generate_local_expert_boolean_mask(local_expert_indices: torch.Tensor, num_experts: int) -> torch.Tensor:
        """``[slots]`` logical ids of this rank's physical slots → ``[E, slots]`` one-hot-per-column boolean map."""
        ids = torch.arange(num_experts, dtype=torch.int32, device=local_expert_indices.device).unsqueeze(1)
        return ids == local_expert_indices.reshape(1, -1).to(torch.int32)

    @staticmethod
    def generate_mask_with_no_local_redundancy(mask: torch.Tensor) -> torch.Tensor:
        """Keep only the FIRST slot of every logical expert that appears more than once on this rank."""
        first = torch.cumsum(mask.to(torch.int32), dim=1) == 1
        return first & mask

    @staticmethod
    def generate_local_expert_id_no_local_redundancy(mask: torch.Tensor, device=None) -> torch.Tensor:
        """``[E, slots]`` map → per-slot logical expert id, ``-1`` for slots masked out as local duplicates."""
        ids = torch.arange(mask.shape[0], dtype=torch.int32, device=mask.device).unsqueeze(1).expand_as(mask)
        return torch.where(mask, ids, torch.full_like(ids, -1)).max(dim=0).values

    def generate_local_expert_mask_with_redundancy(self, local_expert_mask: torch.Tensor, local_expert_indices: torch.Tensor,
                                                   expert_start_ids: torch.Tensor, expert_end_ids: torch.Tensor,
                                                   num_experts: int, rank) -> torch.Tensor:
        """``local_expert_mask [T, slots]`` restricted to the token-position range this rank's replica of each expert is
        responsible for (see :meth:`allocate_token_blocks`), and zeroed for slots that duplicate another local slot."""
        slots = local_expert_indices.reshape(-1).long()
        r = int(rank) if not isinstance(rank, torch.Tensor) else rank.reshape(-1)[0].long()
        lo, hi = expert_start_ids[r, slots][None, :], expert_end_ids[r, slots][None, :]
        pos = torch.arange(local_expert_mask.shape[0], device=local_expert_mask.device)[:, None]
        out = local_expert_mask.masked_fill(~((pos >= lo) & (pos <= hi)), 0)
        uniq = self.generate_local_expert_id_no_local_redundancy(
            self.generate_mask_with_no_local_redundancy(self.generate_local_expert_boolean_mask(slots, num_experts)))
        return out.masked_fill((uniq == -1)[None, :], 0)

    @staticmethod
    def get_block_conditions(block_size: int, num_blocks: int, token_position_to_id: torch.Tensor) -> torch.Tensor:
        """``[num_blocks]`` int32: 1 where a block holds at least one real token (``-1`` = padding) — lets a persistent
        grouped-GEMM kernel skip empty blocks without a host round trip."""
        return (token_position_to_id.view(num_blocks, block_size) != -1).any(dim=1).to(torch.int32)

    def use_index_calc_kernel(self, total_tokens: int) -> bool:
        """Whether the block / token index computation runs as one device pass (always available here: sort + prefix
        sums); the reference's extra shape restrictions do not apply, its config switches are honoured."""
        if self.training or not self.is_prefill or not getattr(self.routed_experts_mlp_config, "use_index_calc_kernel", True):
            return False
        return can_use_find_index_kernel(total_tokens, self.bw.block_size, len(self.local_expert_ids))

    def initialize_mlp_op(self, tensor_model_parallel_group=None, expert_model_parallel_group=None, is_prefill: bool = True):
        """(Re)build the expert weights for the given groups (reference :148-177) and return them."""
        self.mlp_op = self._build_experts(tensor_model_parallel_group, expert_model_parallel_group, is_prefill)
        self.local_expert_ids = self.mlp_op.local_expert_ids
        return self.mlp_op

    def get_blockwise_expert_and_token_mapping_kernel(self, total_tokens: int, num_blocks: int, expert_mask: torch.Tensor,
                                                      expert_index: torch.Tensor, block_size: Optional[int] = None, **kw):
        """Same result as :meth:`get_blockwise_expert_and_token_mapping` (both are device passes here)."""
        return self.get_blockwise_expert_and_token_mapping(total_tokens, num_blocks, expert_mask, expert_index, block_size, **kw)

    # ------------------------------------------------------------------ modes
    def setup_all_experts(self, hidden_states, expert_affinities, expert_index, chosen_expert_indices=None, padding_mask=None):
        num_experts = self.num_experts if chosen_expert_indices is None else len(chosen_expert_indices)
        expert_mask = self.get_expert_mask(expert_index, self.num_experts)
        a = self._topk_affinities(expert_affinities, expert_index, padding_mask)
        if chosen_expert_indices is not None:
            expert_mask, a = expert_mask[:, chosen_expert_indices], a[:, chosen_expert_indices]
        return num_experts, expert_mask, a, hidden_states

    def forward_all_experts(self, hidden_states: torch.Tensor, expert_affinities: torch.Tensor, expert_index: torch.Tensor, chosen_expert_indices=None,
                            padding_mask=None) -> torch.Tensor:
        x, aff, idx = hidden_states, expert_affinities, expert_index      # reference parameter names in the signature
        mlp_op = self.get_mlp_op()
        a = self._topk_affinities(aff, idx, padding_mask)                     # [T, E]
        local = torch.as_tensor(mlp_op.local_expert_ids, device=x.device)
        if chosen_expert_indices is not None:
            local = local[chosen_expert_indices]
        w = a[:, local].t().unsqueeze(-1)                                     # [E_l, T, 1]
        xe = x.unsqueeze(0).expand(local.numel(), *x.shape)                   # [E_l, T, H]
        if self.cfg.early_expert_affinity_modulation:
            y = mlp_op(xe * w.to(x.dtype), chosen_expert_indices)             # scale the expert INPUT, mask the output
            return (y * (w > 0).to(y.dtype)).sum(0)
        y = mlp_op(xe, chosen_expert_indices)                                 # [E_l, T, H]
        return (y * w.to(y.dtype)).sum(0)

    def forward_all_experts_EP(self, hidden_states: torch.Tensor, expert_affinities: torch.Tensor, expert_index: torch.Tensor,
                               chosen_expert_indices=None, padding_mask=None) -> torch.Tensor:
        """Inference EP: every rank runs its local experts on all tokens; the MoE layer sums over the EP group."""
        x, aff, idx = hidden_states, expert_affinities, expert_index      # reference parameter names in the signature
        return self.forward_all_experts(x, aff, idx, padding_mask=padding_mask)

    def forward_selective_loading(self, hidden_states: torch.Tensor, expert_affinities: torch.Tensor, expert_index: torch.Tensor) -> torch.Tensor:
        """Touch only the ``T·k`` chosen experts (decode / short speculation windows, reference :595-625).  Vectorised
        over tokens: the (token, slot) pairs become ``T·k`` single-token "experts" of one batched contraction."""
        x, aff, idx = hidden_states, expert_affinities, expert_index      # reference parameter names in the signature
        if self.ep > 1:
            raise NotImplementedError("Selective Loading with Expert parallelism is not supported in token generation.")
        mlp_op = self.get_mlp_op()
        T, k = idx.shape
        chosen = aff.gather(1, idx)                                           # [T, k]
        if self.cfg.normalize_top_k_affinities:
            chosen = chosen / chosen.abs().sum(-1, keepdim=True).clamp(min=1e-12)
        flat_e = idx.reshape(-1)                                              # [T·k]
        xin = x.repeat_interleave(k, 0).unsqueeze(1)                          # [T·k, 1, H]
        w = chosen.reshape(-1, 1, 1)
        if self.cfg.early_expert_affinity_modulation:
            y = mlp_op(xin * w.to(x.dtype), flat_e)
        else:
            y = mlp_op(xin, flat_e)
            y = y * w.to(y.dtype)
        return y.reshape(T, k, -1).sum(1)

    def forward_capacity_factor(self, hidden_states: torch.Tensor, expert_affinities: torch.Tensor, expert_index: torch.Tensor, padding_mask=None) -> torch.Tensor:
        x, aff, idx = hidden_states, expert_affinities, expert_index      # reference parameter names in the signature
        T, H = x.shape
        E, k = self.num_experts, self.top_k
        cf = self.capacity_factor if self.capacity_factor is not None else E / k
        C = min(T, max(1, math.ceil(cf * T * k / E)))
        a = self._topk_affinities(aff, idx, padding_mask)
        # position of every (token, slot) inside its expert's queue, in slot-major routing order
        onehot = torch.zeros(k, T, E, dtype=torch.long, device=x.device)
        onehot.scatter_(2, idx.t().unsqueeze(-1), 1)
        if padding_mask is not None:
            onehot = onehot * padding_mask.reshape(1, -1, 1).long()           # padded tokens take no capacity
        flat = onehot.reshape(k * T, E)
        pos = (torch.cumsum(flat, dim=0) - 1) * flat                           # [k·T, E]
        keep = (flat == 1) & (pos < C)
        pos = pos.reshape(k, T, E)
        keep = keep.reshape(k, T, E)
        keep_te = keep.any(0)                                                  # [T, E]
        pos_te = (pos * keep.long()).sum(0)                                    # [T, E]
        # dispatch: [E, C, H]
        disp = torch.zeros(E, C, H, dtype=x.dtype, device=x.device)
        t_idx, e_idx = keep_te.nonzero(as_tuple=True)
        early = self.cfg.early_expert_affinity_modulation
        src = x[t_idx] * a[t_idx, e_idx].unsqueeze(-1).to(x.dtype) if early else x[t_idx]
        disp[e_idx, pos_te[t_idx, e_idx]] = src
        mlp_op = self.get_mlp_op()
        if self.ep > 1 and self.training:
            d = mappings.enter_expert_parallel_region(disp, scatter_gather=False)        # [E/ep, ep, C, H]
            e_l, ep, _, _ = d.shape
            y = mlp_op(d.reshape(e_l, ep * C, H)).reshape(e_l, ep, C, H)
            y = mappings.exit_expert_parallel_region(y, scatter_gather=False)            # [E, C, H]
        else:
            local = torch.as_tensor(mlp_op.local_expert_ids, device=x.device)
            y_l = mlp_op(disp[local])
            y = torch.zeros(E, C, H, dtype=y_l.dtype, device=x.device)
            y[local] = y_l
        out = torch.zeros(T, H, dtype=y.dtype, device=x.device)
        picked = y[e_idx, pos_te[t_idx, e_idx]]
        out.index_add_(0, t_idx, picked if early else picked * a[t_idx, e_idx].unsqueeze(-1).to(y.dtype))
        return out

    def forward_blockwise(self, hidden_states: torch.Tensor, expert_affinities: torch.Tensor, expert_index: torch.Tensor, expert_affinities_masked_full=None,
                          padding_mask=None) -> torch.Tensor:
        x, aff, idx = hidden_states, expert_affinities, expert_index      # reference parameter names in the signature
        a = expert_affinities_masked_full if expert_affinities_masked_full is not None else \
            self._topk_affinities(aff, idx, padding_mask)
        if self.ep > 1:
            # inference-style EP: routing masked to the experts this rank owns, results are summed over EP by the caller
            return self.forward_all_experts(x, aff, idx, padding_mask=padding_mask)
        if self.cfg.early_expert_affinity_modulation or self.cfg.bias:
            return self.forward_all_experts(x, aff, idx, padding_mask=padding_mask)     # the grouped path scales outputs only
        return blockwise_expert_mlp(x, a, idx, self.get_mlp_op(), min(self.bw.block_size, max(16, x.shape[0])))

    def torch_blockwise_matmul_inference(self, hidden_states, expert_affinities_masked, expert_index, **_unused):
        """PyTorch form of the dropless computation on pre-masked affinities (reference :1350-1405)."""
        return blockwise_expert_mlp(hidden_states, expert_affinities_masked, expert_index, self.get_mlp_op(),
                                    min(self.bw.block_size, max(16, hidden_states.shape[0])))

    def forward(self, hidden_states: torch.Tensor, expert_affinities: torch.Tensor, expert_index: torch.Tensor,
                seq_len: Optional[int] = None, padding_mask: Optional[torch.Tensor] = None,
                expert_affinities_masked_full: Optional[torch.Tensor] = None) -> torch.Tensor:
        """hidden ``[T, H]`` (already gathered over SP), affinities ``[T, E]``, index ``[T, k]`` → ``[T, H]`` partial sums
        over TP (and EP) — the MoE layer performs the delayed reduction."""
        x = hidden_states.reshape(-1, hidden_states.shape[-1])
        T, c = x.shape[0], self.routed_experts_mlp_config
        self._decode_hint = (not self.training) and seq_len == 1
        dense_enough = T * self.top_k >= self.bw.block_size or T * self.top_k > self.num_experts * 4
        if self.training:
            if c.capacity_factor is not None and c.capacity_factor > 0:
                out = self.forward_capacity_factor(x, expert_affinities, expert_index, padding_mask)
            elif dense_enough and self.ep == 1 and c.glu_mlp:
                out = self.forward_blockwise(x, expert_affinities, expert_index, None, padding_mask)
            elif self.ep > 1:
                out = self.forward_capacity_factor(x, expert_affinities, expert_index, padding_mask)   # full capacity via all-to-all
            else:
                out = self.forward_all_experts(x, expert_affinities, expert_index, padding_mask=padding_mask)
        else:
            frac_loaded = T * self.top_k / self.num_experts
            selective = frac_loaded < DEFAULT_SELECTIVE_LOADING_THRESHOLD and self.ep == 1 and padding_mask is None \
                and seq_len is not None
            if seq_len == 1:
                out = self.forward_selective_loading(x, expert_affinities, expert_index) if selective else \
                    (self.forward_all_experts_EP if self.ep > 1 else self.forward_all_experts)(
                        x, expert_affinities, expert_index, padding_mask=padding_mask)
            elif c.capacity_factor is not None and c.capacity_factor > 0 and self.ep == 1:
                out = self.forward_capacity_factor(x, expert_affinities, expert_index, padding_mask)
            elif selective:
                out = self.forward_selective_loading(x, expert_affinities, expert_index)
            elif not dense_enough or self.ep > 1:
                out = self.forward_all_experts(x, expert_affinities, expert_index, padding_mask=padding_mask)
            else:
                out = self.forward_blockwise(x, expert_affinities, expert_index, expert_affinities_masked_full, padding_mask)
        return out.view(hidden_states.shape)




def create_spmd_ranks(model_state_dict, prefix: str, world_size: int, n_routed_experts: Optional[int] = None,
                      expert_model_parallel_group=None, spmd_rank_name: str = "spmd_rank", expert_distribution=None) -> None:
    """Reference :1501-1530 — add ``{prefix}{spmd_rank_name}.rank = arange(world)`` to a full checkpoint and, with expert
    parallelism, ``….local_expert_indices`` ``[world, experts per EP rank]``: the logical experts every global rank hosts
    (contiguous blocks, or ``expert_distribution[ep_rank]`` when experts are placed explicitly / redundantly)."""
    model_state_dict[f"{prefix}{spmd_rank_name}.rank"] = torch.arange(0, world_size, dtype=torch.int32)
    ep = 1 if expert_model_parallel_group is None else (
        expert_model_parallel_group.size() if hasattr(expert_model_parallel_group, "size") else int(expert_model_parallel_group))
    if ep > 1:
        assert n_routed_experts is not None, "n_routed_experts is required with expert parallelism"
        rows = []
        for rank in range(world_size):
            ep_rank = ps.get_expert_parallel_rank_from_global_rank(rank, expert_model_parallel_group)
            rows.append(ps.get_experts_for_expert_parallel_rank(ep_rank, total_number_of_experts=n_routed_experts,
                                                                expert_model_parallel_size=ep,
                                                                expert_distribution=expert_distribution))
        model_state_dict[f"{prefix}{spmd_rank_name}.local_expert_indices"] = torch.tensor(rows, dtype=torch.int32)


def duplicate_and_replace_prefixes(old_prefix: str, new_prefix: str, model_state_dict) -> None:
    """Hybrid sharding: alias every ``…old_prefix…`` entry under ``…new_prefix…`` so the same full tensor can be cut with a
    second sharding strategy (reference :1532-1546)."""
    for key in [k for k in model_state_dict if old_prefix in k]:
        model_state_dict[key.replace(old_prefix, new_prefix)] = model_state_dict[key]


def can_use_find_index_kernel(T: int, block_size: int, E_local: int, logical_nc_config: int = 1, tp_size: int = 1,
                              ep_size: int = 1) -> bool:
    """Whether the on-device block/token index computation applies.  The reference's NKI kernel has shape constraints
    (:1549-1590); ``blockwise.build_block_metadata`` (sort + prefix sums, no host sync) has none beyond a positive
    block size, so this only rejects degenerate input."""
    return T > 0 and block_size > 0 and E_local > 0
