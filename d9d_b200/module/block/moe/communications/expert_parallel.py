from __future__ import annotations

from typing import Any

import torch
import torch.distributed as dist
from torch.autograd import Function

from d9d_b200.kernel.moe import MoELayout, build_moe_layout, moe_permute, moe_unpermute

from .base import ExpertCommunicationHandler


class _ExchangeRows(Function):
    """Variable-split all-to-all of leading-dim rows; the backward is the same exchange with the splits swapped."""

    @staticmethod
    def forward(ctx: Any, rows: torch.Tensor, send_splits: list[int], recv_splits: list[int], group: dist.ProcessGroup):
        ctx.send_splits, ctx.recv_splits, ctx.group = send_splits, recv_splits, group
        out = rows.new_empty((sum(recv_splits), *rows.shape[1:]))
        dist.all_to_all_single(out, rows.contiguous(), recv_splits, send_splits, group=group)
        return out

    @staticmethod
    def backward(ctx: Any, grad: torch.Tensor):  # type: ignore[override]
        out = grad.new_empty((sum(ctx.send_splits), *grad.shape[1:]))
        dist.all_to_all_single(out, grad.contiguous(), ctx.send_splits, ctx.recv_splits, group=ctx.group)
        return out, None, None, None


def _exchange(rows: torch.Tensor, send_splits: list[int], recv_splits: list[int], group: dist.ProcessGroup) -> torch.Tensor:
    return _ExchangeRows.apply(rows, send_splits, recv_splits, group)


class ExpertParallelCommunicationHandler(ExpertCommunicationHandler):
    """Expert-parallel dispatch/combine: every rank of ``group`` owns ``num_experts / group.size()`` experts.

    Plays the role of the reference's DeepEP handler (``moe/communications/deepep.py:57-222``) without the external
    library:

    1. (token, slot) pairs are stable-sorted by *global* expert id with the device-side counting sort in compact
       (``align=1``) mode – that order is grouped by destination rank and, inside a rank, by local expert;
    2. per-expert counts are exchanged (one small all-to-all), then rows, routing probabilities and local expert
       ids travel with one variable-split all-to-all each;
    3. the receiver builds a 128-row aligned :class:`MoELayout` over what it received (rows arrive ordered by
       source rank, the layout regroups them by local expert) and the grouped wgmma GEMMs consume it directly;
    4. ``combine`` walks the same path backwards and sums each token's ``top_k`` partial outputs in fp32.

    The only host synchronisation is the read of the split sizes that NCCL's all-to-all needs.
    """

    def __init__(self, num_experts: int):
        self._num_experts = num_experts
        self._group: dist.ProcessGroup | None = None
        self._state: tuple[MoELayout, MoELayout, list[int], list[int]] | None = None

    def setup(self, group: dist.ProcessGroup, hidden_size: int, hidden_dtype: torch.dtype) -> None:
        if self._num_experts % group.size() != 0:
            raise ValueError(f"{self._num_experts} experts cannot be split across {group.size()} expert-parallel ranks")
        self._group = group
        self._hidden_size = hidden_size
        self._hidden_dtype = hidden_dtype

    @property
    def num_local_experts(self) -> int:
        assert self._group is not None
        return self._num_experts // self._group.size()

    def dispatch(self, hidden_states: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor):
        group = self._group
        if group is None:
            raise ValueError("ExpertParallelCommunicationHandler.setup() was not called")
        ranks = group.size()
        local_experts = self.num_local_experts

        send_layout = build_moe_layout(topk_ids, self._num_experts, align=1)
        send_counts = send_layout.counts  # [E] int32, rows per global expert == per (destination rank, local expert)
        recv_counts = torch.empty_like(send_counts)  # [ranks, local_experts]: rows from every source rank
        dist.all_to_all_single(recv_counts, send_counts, group=group)
        splits = torch.stack([send_counts.view(ranks, local_experts).sum(1), recv_counts.view(ranks, local_experts).sum(1)])
        send_splits, recv_splits = splits.tolist()  # the one host sync of the layer

        send_x, send_p = moe_permute(hidden_states, topk_weights, send_layout)
        expert_of_row = torch.repeat_interleave(
            torch.arange(self._num_experts, device=topk_ids.device, dtype=torch.int64) % local_experts,
            send_counts.long(), output_size=send_layout.capacity)

        recv_x = _exchange(send_x, send_splits, recv_splits, group)
        recv_p = _exchange(send_p, send_splits, recv_splits, group)
        recv_e = _exchange(expert_of_row, send_splits, recv_splits, group)

        recv_layout = build_moe_layout(recv_e[:, None], local_experts)
        xp, pp = moe_permute(recv_x, recv_p[:, None], recv_layout)
        self._state = (send_layout, recv_layout, send_splits, recv_splits)
        return xp, pp, recv_layout

    def combine(self, hidden_states: torch.Tensor) -> torch.Tensor:
        if self._state is None or self._group is None:
            raise ValueError("Cannot run combine before running dispatch!")
        send_layout, recv_layout, send_splits, recv_splits = self._state
        self._state = None
        received_order = moe_unpermute(hidden_states, recv_layout)
        sent_order = _exchange(received_order, recv_splits, send_splits, self._group)
        return moe_unpermute(sent_order, send_layout)
