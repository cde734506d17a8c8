from __future__ import annotations

import torch
from torch import nn
from torch.distributed import ProcessGroup

from d9d_b200.module.base import ModuleLateInit

from .communications import ExpertCommunicationHandler, NoCommunicationHandler
from .grouped_experts import GroupedSwiGLU
from .router import RouterParameters, TopKRouter
from .shared_expert import SharedExpertParameters, SharedSwiGLU


class MoELayer(nn.Module, ModuleLateInit):
    """Router -> dispatch -> grouped experts -> combine (+ optional shared expert).

    Parity: reference ``d9d/module/block/moe/layer.py:16-141``.
    """

    def __init__(self, hidden_dim: int, intermediate_dim_grouped: int, num_grouped_experts: int, top_k: int,
                 router_renormalize_probabilities: bool, shared_expert: SharedExpertParameters | None = None,
                 router: RouterParameters | None = None):
        super().__init__()
        self.router = TopKRouter(dim=hidden_dim, num_experts=num_grouped_experts, top_k=top_k,
                                 renormalize_probabilities=router_renormalize_probabilities, options=router)
        self.grouped_experts = GroupedSwiGLU(hidden_dim=hidden_dim, intermediate_dim=intermediate_dim_grouped,
                                             num_experts=num_grouped_experts)
        self.shared_expert = SharedSwiGLU(hidden_size=hidden_dim, params=shared_expert) if shared_expert is not None else None
        self._communicator: ExpertCommunicationHandler = NoCommunicationHandler(num_grouped_experts)
        self._num_grouped_experts = num_grouped_experts
        self._hidden_dim = hidden_dim
        self.tokens_per_expert = nn.Buffer(torch.empty((num_grouped_experts,), dtype=torch.int64), persistent=False)

    def enable_distributed_communicator(self, group: ProcessGroup) -> None:
        """Switch to expert-parallel dispatch/combine over ``group`` (NVLink peer memory / NCCL all-to-all)."""
        from .communications.nvlink import AutoExpertParallelCommunicationHandler  # lazy: needs a process group

        handler = AutoExpertParallelCommunicationHandler(num_experts=self._num_grouped_experts)
        handler.setup(group, self._hidden_dim, self.router.gate.weight.dtype)
        self._communicator = handler

    @torch.no_grad()
    def _update_tokens_per_expert(self, expert_indices: torch.Tensor) -> None:
        flat = expert_indices.reshape(-1)
        self.tokens_per_expert.scatter_add_(0, flat, torch.ones_like(flat, dtype=self.tokens_per_expert.dtype))

    @torch.no_grad()
    def reset_stats(self) -> None:
        self.tokens_per_expert.zero_()

    def forward(self, hidden_states: torch.Tensor) -> torch.Tensor:
        shape = hidden_states.shape
        x = hidden_states.reshape(-1, shape[-1])
        shared = self.shared_expert(x) if self.shared_expert is not None else None

        seq = {}
        if self.router.sequence_balance_coef > 0:
            if hidden_states.dim() != 3:
                raise ValueError("the sequence-wise balance loss needs the MoE input as [batch, sequence, hidden], got "
                                 f"{tuple(shape)}")
            seq = {"sequence_length": shape[-2]}
        routing = self.router(x, **seq)
        self._update_tokens_per_expert(routing.selected_expert_indices)

        xp, pp, grouping = self._communicator.dispatch(x, routing.selected_expert_indices, routing.selected_probabilities)
        out_buf, dx_buf = self._communicator.expert_buffers()
        yp = self.grouped_experts(xp, pp, grouping, out=out_buf, dx_out=dx_buf)
        y = self._communicator.combine(yp)
        if shared is not None:
            y = y + shared
        return y.reshape(shape)

    def reset_parameters(self) -> None:
        self.router.reset_parameters()
        self.grouped_experts.reset_parameters()
        if self.shared_expert is not None:
            self.shared_expert.reset_parameters()
        nn.init.zeros_(self.tokens_per_expert)
