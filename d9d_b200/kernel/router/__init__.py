"""Fused MoE routing: fp32 softmax or sigmoid scores + top-k (+ selection bias, + group-limited selection, + renormalisation,
+ scaling) and its backward."""

from __future__ import annotations

from typing import Any

import torch
import torch.nn.functional as F
from torch.autograd import Function

from .._native import native_ops, on_gpu


def route_topk_reference(logits: torch.Tensor, top_k: int, renormalize: bool, expert_bias: torch.Tensor | None = None):
    """Plain PyTorch definition (CPU path and numerics oracle): returns ``(indices [T,k] int64, probs [T,k] fp32)``."""
    probs = F.softmax(logits, dim=-1, dtype=torch.float32)
    if expert_bias is None:
        chosen_p, chosen = torch.topk(probs, k=top_k, dim=-1)
    else:
        chosen = torch.topk(probs + expert_bias, k=top_k, dim=-1).indices
        chosen_p = probs.gather(-1, chosen)
    if renormalize:
        chosen_p = chosen_p / (chosen_p.sum(dim=-1, keepdim=True) + 1e-20)
    return chosen, chosen_p


class _RouteTopK(Function):
    @staticmethod
    def forward(ctx: Any, logits: torch.Tensor, top_k: int, renormalize: bool, expert_bias: torch.Tensor | None,
                score_function: str, num_groups: int, topk_groups: int, scaling_factor: float):
        idx, probs = native_ops().router_topk_fwd(logits, expert_bias, top_k, renormalize, score_function, num_groups,
                                                  topk_groups, scaling_factor)
        ctx.save_for_backward(logits, idx)
        ctx.renormalize = renormalize
        ctx.score_function = score_function
        ctx.scaling_factor = scaling_factor
        ctx.mark_non_differentiable(idx)
        return idx, probs

    @staticmethod
    def backward(ctx: Any, _didx: torch.Tensor, dprobs: torch.Tensor):  # type: ignore[override]
        logits, idx = ctx.saved_tensors
        dlogits = native_ops().router_topk_bwd(logits, idx, dprobs.float().contiguous(), ctx.renormalize, ctx.score_function,
                                               ctx.scaling_factor)
        return dlogits, None, None, None, None, None, None, None


def route_topk_general(logits: torch.Tensor, top_k: int, renormalize: bool, expert_bias: torch.Tensor | None = None,
                       score_function: str = "softmax", num_groups: int = 1, topk_groups: int = 1, scaling_factor: float = 1.0):
    """DeepSeek-style routing in plain PyTorch (differentiable through the selected scores).

    ``score_function``: ``softmax`` over all experts or independent ``sigmoid`` scores.  Selection uses ``score + expert_bias``
    (auxiliary-loss-free balancing), mixing weights use the unbiased scores.  With ``num_groups > 1`` experts are split into
    equal groups, only the ``topk_groups`` best groups stay eligible (group score: sum of the group's two best selection
    scores - DeepSeek-V3 - or, for a single-expert comparison, its best one when groups hold one expert).  Finally the ``k``
    weights are optionally renormalised to sum to one and multiplied by ``scaling_factor``.
    """
    if score_function == "softmax":
        scores = F.softmax(logits, dim=-1, dtype=torch.float32)
    elif score_function == "sigmoid":
        scores = torch.sigmoid(logits.float())
    else:
        raise ValueError(f"unknown router score function {score_function!r}")
    choice = scores if expert_bias is None else scores + expert_bias
    num_experts = logits.shape[-1]
    if num_groups > 1:
        if num_experts % num_groups != 0 or not 0 < topk_groups <= num_groups:
            raise ValueError("experts must split evenly into groups and 0 < topk_groups <= num_groups")
        per_group = choice.reshape(*choice.shape[:-1], num_groups, num_experts // num_groups)
        group_scores = per_group.topk(min(2, per_group.shape[-1]), dim=-1).values.sum(dim=-1)
        keep = torch.zeros_like(group_scores, dtype=torch.bool).scatter_(-1, group_scores.topk(topk_groups, dim=-1).indices, True)
        choice = per_group.masked_fill(~keep.unsqueeze(-1), 0.0).reshape(choice.shape)
    chosen = torch.topk(choice.detach(), k=top_k, dim=-1).indices
    chosen_p = scores.gather(-1, chosen)
    if renormalize:
        chosen_p = chosen_p / (chosen_p.sum(dim=-1, keepdim=True) + 1e-20)
    if scaling_factor != 1.0:
        chosen_p = chosen_p * scaling_factor
    return chosen, chosen_p


def route_topk(logits: torch.Tensor, top_k: int, renormalize: bool, expert_bias: torch.Tensor | None = None,
               score_function: str = "softmax", num_groups: int = 1, topk_groups: int = 1, scaling_factor: float = 1.0):
    """``logits [..., E]`` -> ``(indices [..., k] int64, probabilities [..., k] fp32)``.

    bf16 CUDA logits with ``E <= 1024``, ``k <= min(32, E)`` and at most 32 expert groups run on the fused CUDA kernel,
    whatever the routing options (softmax or sigmoid scores, bias, group-limited selection, renormalisation, scaling).
    Other inputs use the PyTorch definitions: ``route_topk_reference`` for plain softmax top-k, ``route_topk_general``
    for the DeepSeek variants.
    """
    num_experts = logits.shape[-1]
    if num_groups > 1 and (num_experts % num_groups != 0 or not 0 < topk_groups <= num_groups):
        raise ValueError("experts must split evenly into groups and 0 < topk_groups <= num_groups")
    if score_function not in ("softmax", "sigmoid"):
        raise ValueError(f"unknown router score function {score_function!r}")
    if (on_gpu(logits) and logits.dtype == torch.bfloat16 and num_experts <= 1024 and top_k <= min(32, num_experts)
            and num_groups <= 32):
        flat = logits.reshape(logits.shape[:-1].numel(), num_experts)  # also when there are no tokens
        if not flat.is_contiguous():
            flat = flat.contiguous()
        groups = (num_groups, topk_groups) if num_groups > 1 else (1, 1)
        idx, probs = _RouteTopK.apply(flat, top_k, renormalize, None if expert_bias is None else expert_bias.float().contiguous(),
                                      score_function, *groups, float(scaling_factor))
        return idx.view(*logits.shape[:-1], top_k), probs.view(*logits.shape[:-1], top_k)
    if score_function != "softmax" or num_groups > 1 or scaling_factor != 1.0:
        return route_topk_general(logits, top_k, renormalize, expert_bias, score_function, num_groups, topk_groups, scaling_factor)
    return route_topk_reference(logits, top_k, renormalize, expert_bias)


__all__ = ["route_topk", "route_topk_general", "route_topk_reference"]
