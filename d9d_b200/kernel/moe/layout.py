from __future__ import annotations

import dataclasses
from typing import Any

import torch
from torch.autograd import Function

from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection

from .._native import contiguous_aligned, fused_wgrad_buffer, fused_wgrad_owner, grad_dtype_of, native_ops, on_gpu

ALIGN = 128  # GEMM BLOCK_M: expert segments never share an M-tile, per-expert K ranges are BLOCK_K aligned


@dataclasses.dataclass
class MoELayout:
    """Device-resident description of the expert-sorted, 128-row aligned token layout."""

    counts: torch.Tensor  # [E] int32 tokens per expert
    seg_offsets: torch.Tensor  # [E+1] int32 aligned segment starts
    row_map: torch.Tensor  # [T*k] int32 destination row of every (token, slot) or -1
    tile_group: torch.Tensor  # [capacity/128] int32 expert of every row tile or -1
    num_tokens: int
    top_k: int
    num_experts: int
    capacity: int  # static upper bound on rows (T*k + E*(align-1) rounded up)
    align: int = ALIGN  # 128 for GEMM-ready layouts, 1 for the compact send order of the expert-parallel all-to-all


def layout_capacity(num_tokens: int, top_k: int, num_experts: int, align: int = ALIGN) -> int:
    n = num_tokens * top_k + num_experts * (align - 1)
    return (n + align - 1) // align * align


def _build_layout_reference(topk_ids: torch.Tensor, num_experts: int, capacity: int, align: int = ALIGN):
    flat = topk_ids.reshape(-1)
    valid = (flat >= 0) & (flat < num_experts)
    counts = torch.bincount(flat[valid], minlength=num_experts)
    aligned = (counts + align - 1) // align * align
    seg = torch.zeros(num_experts + 1, dtype=torch.long, device=flat.device)
    seg[1:] = aligned.cumsum(0)
    key = torch.where(valid, flat, torch.full_like(flat, num_experts))
    order = torch.sort(key, stable=True).indices
    sorted_key = key[order]
    first = torch.searchsorted(sorted_key, torch.arange(num_experts + 1, device=flat.device))
    rank = torch.arange(flat.numel(), device=flat.device) - first[sorted_key.clamp_max(num_experts)]
    dest_sorted = torch.where(sorted_key < num_experts, seg[sorted_key.clamp_max(num_experts - 1)] + rank, torch.full_like(rank, -1))
    row_map = torch.empty_like(flat)
    row_map[order] = dest_sorted
    num_tiles = capacity // ALIGN if align % ALIGN == 0 else 0
    tiles = torch.full((num_tiles,), -1, dtype=torch.long, device=flat.device)
    tile_idx = torch.arange(num_tiles, device=flat.device) * ALIGN
    owner = torch.searchsorted(seg, tile_idx, right=True) - 1
    used = tile_idx < seg[-1]
    tiles[used] = owner[used]
    return counts.int(), seg.int(), row_map.int(), tiles.int()


def build_moe_layout(topk_ids: torch.Tensor, num_experts: int, align: int = ALIGN) -> MoELayout:
    """``topk_ids [T, k]`` (ids outside ``[0, E)`` are dropped) -> layout. No host synchronisation.

    ``align=128`` gives the GEMM-ready layout; ``align=1`` a compact stable sort by expert (used as the send order
    of the expert-parallel exchange, where padding would waste NVLink bandwidth).
    """
    T, k = topk_ids.shape
    cap = layout_capacity(T, k, num_experts, align)
    ids = topk_ids.contiguous()
    if ids.dtype != torch.int64:
        ids = ids.long()
    if on_gpu(ids):
        counts, seg, row_map, tile_group = native_ops().moe_build_layout(ids, num_experts, align, cap)
    else:
        counts, seg, row_map, tile_group = _build_layout_reference(ids, num_experts, cap, align)
    return MoELayout(counts, seg, row_map, tile_group, T, k, num_experts, cap, align)


# ------------------------------------------------------------------------------------------ permute / unpermute
def _scatter_reference(x: torch.Tensor, probs: torch.Tensor | None, layout: MoELayout):
    rm = layout.row_map.long()
    valid = rm >= 0
    tok = torch.arange(layout.num_tokens, device=x.device).repeat_interleave(layout.top_k)
    xp = x.new_zeros(layout.capacity, x.shape[1])
    xp[rm[valid]] = x[tok[valid]]
    pp = None
    if probs is not None:
        pp = torch.zeros(layout.capacity, dtype=torch.float32, device=x.device)
        pp[rm[valid]] = probs.reshape(-1).float()[valid]
    return xp, pp


def _gather_reference(yp: torch.Tensor, dpp: torch.Tensor | None, layout: MoELayout):
    rm = layout.row_map.long()
    valid = rm >= 0
    tok = torch.arange(layout.num_tokens, device=yp.device).repeat_interleave(layout.top_k)
    y = torch.zeros(layout.num_tokens, yp.shape[1], dtype=torch.float32, device=yp.device)
    y.index_add_(0, tok[valid], yp[rm[valid]].float())
    dprobs = None
    if dpp is not None:
        dprobs = torch.zeros(layout.num_tokens * layout.top_k, dtype=torch.float32, device=yp.device)
        dprobs[valid] = dpp[rm[valid]]
        dprobs = dprobs.view(layout.num_tokens, layout.top_k)
    return y.to(yp.dtype), dprobs


def _scatter(x, probs, layout: MoELayout):
    if on_gpu(x):
        xp, pp = native_ops().moe_permute(contiguous_aligned(x), None if probs is None else probs.float().contiguous(),
                                          layout.row_map, layout.counts, layout.seg_offsets, layout.capacity)
        return xp, (pp if probs is not None else None)
    return _scatter_reference(x, probs, layout)


def _gather(yp, dpp, layout: MoELayout):
    if on_gpu(yp):
        y, dprobs = native_ops().moe_gather(contiguous_aligned(yp), None if dpp is None else dpp.contiguous(), layout.row_map,
                                            layout.num_tokens, layout.top_k)
        return y, (dprobs if dpp is not None else None)
    return _gather_reference(yp, dpp, layout)


class _PermuteFunction(Function):
    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, probs: torch.Tensor, layout: MoELayout):
        ctx.layout = layout
        ctx.probs_dtype = probs.dtype
        xp, pp = _scatter(x, probs, layout)
        return xp, pp

    @staticmethod
    def backward(ctx: Any, dxp: torch.Tensor, dpp: torch.Tensor):  # type: ignore[override]
        dx, dprobs = _gather(dxp, dpp.float() if dpp is not None else None, ctx.layout)
        return dx, (dprobs.to(ctx.probs_dtype) if dprobs is not None else None), None


class _UnpermuteFunction(Function):
    @staticmethod
    def forward(ctx: Any, yp: torch.Tensor, layout: MoELayout):
        ctx.layout = layout
        y, _ = _gather(yp, None, layout)
        return y

    @staticmethod
    def backward(ctx: Any, dy: torch.Tensor):  # type: ignore[override]
        dyp, _ = _scatter(dy.contiguous(), None, ctx.layout)
        return dyp, None


def moe_permute(x: torch.Tensor, probs: torch.Tensor, layout: MoELayout) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [T,H]``, ``probs [T,k]`` -> expert-sorted ``xp [capacity,H]``, ``pp [capacity]`` (fp32). Pad rows are 0."""
    return _PermuteFunction.apply(x, probs, layout)


def moe_unpermute(yp: torch.Tensor, layout: MoELayout) -> torch.Tensor:
    """``y[t] = sum_j yp[row(t, j)]`` accumulated in fp32."""
    return _UnpermuteFunction.apply(yp, layout)


# ------------------------------------------------------------------------------------------ grouped linear
def _grouped_linear_reference(xp: torch.Tensor, weight: torch.Tensor, layout: MoELayout) -> torch.Tensor:
    out = xp.new_zeros(xp.shape[0], weight.shape[2])
    seg = layout.seg_offsets.tolist()
    for e in range(layout.num_experts):
        if seg[e + 1] > seg[e]:
            out[seg[e] : seg[e + 1]] = xp[seg[e] : seg[e + 1]] @ weight[e]
    return out


class _GroupedLinearFunction(Function):
    @staticmethod
    def forward(ctx: Any, xp: torch.Tensor, weight: torch.Tensor, layout: MoELayout, owner: torch.Tensor | None = None):
        ctx.layout = layout
        ctx.owner = owner  # see ``fused_wgrad_owner``: dW accumulates straight into owner.grad
        ctx.save_for_backward(xp, weight)
        out = torch.empty(xp.shape[0], weight.shape[2], device=xp.device, dtype=xp.dtype)
        native_ops().gemm_grouped_m(xp, weight, out, layout.tile_group, True)
        return out

    @staticmethod
    def backward(ctx: Any, dy: torch.Tensor):  # type: ignore[override]
        xp, weight = ctx.saved_tensors
        layout: MoELayout = ctx.layout
        ops = native_ops()
        dy = dy.contiguous()
        dx = dw = None
        if ctx.needs_input_grad[0] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.inputs):
            dx = torch.empty_like(xp)
            ops.gemm_grouped_m(dy, weight, dx, layout.tile_group, False)  # W[e] read as [N'=in, K'=out]
        if GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.weight):
            if ctx.owner is not None and ctx.needs_input_grad[3]:
                ops.gemm_grouped_k(xp, dy, fused_wgrad_buffer(ctx.owner), layout.seg_offsets, True)  # grad[e] += xp_e^T @ dy_e
            elif ctx.needs_input_grad[1]:
                dw = torch.empty(weight.shape, device=weight.device, dtype=grad_dtype_of(weight))
                ops.gemm_grouped_k(xp, dy, dw, layout.seg_offsets, False)
        return dx, dw, None, None


def grouped_linear(xp: torch.Tensor, weight: torch.Tensor, layout: MoELayout) -> torch.Tensor:
    """``out[r] = xp[r] @ weight[expert(r)]`` with ``weight [E, in, out]`` over the aligned layout.

    NOTE: rows past the last expert segment are left uninitialised (they are never read back).
    """
    if on_gpu(xp):
        owner = fused_wgrad_owner(weight)
        if owner is None:
            return _GroupedLinearFunction.apply(xp, weight, layout, None)
        return _GroupedLinearFunction.apply(xp, weight.detach(), layout, owner)
    return _grouped_linear_reference(xp, weight, layout)
