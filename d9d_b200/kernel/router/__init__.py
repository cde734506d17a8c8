"""Fused MoE routing: fp32 softmax or sigmoid scores + top-k (+ selection bias, + group-limited selection, + renormalisation,
+ scaling) and its backward, optionally with the router's auxiliary losses folded into that backward.

Auxiliary losses of one call (``T`` tokens, ``E`` experts, top-``k``, ``s = softmax(logits)`` in fp32 - unbiased, not
renormalised, not scaled - and ``c_e`` the number of the ``T k`` selections that went to expert ``e``):

* load balancing (Switch Transformer): ``A = E sum_e f_e P_e`` with ``f_e = c_e / (k T)`` (no gradient) and
  ``P_e = mean_t s[t, e]``; 1 when balanced, up to ``E / k`` when every token picks the same ``k`` experts;
* router z-loss (ST-MoE): ``Z = mean_t lse_t^2`` with ``lse_t = logsumexp_e logits[t, e]``.

With ``w`` the loss weight per token, the call's auxiliary objective ``w T (coef_lb A + coef_z Z)`` is back-propagated by
adding its gradient to the logits' gradient in backward, and ``(w T A, w T Z, w T)`` is added to an optional fp32 ``[3]``
accumulator there - once per call, even when activation recomputation runs the forward twice.

Sequence-wise balance loss (DeepSeek-V3 eqs. 17-20, DeepSeek-V2's ``seq_aux``; softmax or sigmoid scores): the ``T`` tokens
are ``B = T / S`` sequences of ``S`` consecutive tokens, ``s[t]`` is the unbiased, unrenormalised, unscaled balance score
(softmax: ``softmax(x_t)``; sigmoid: ``sigmoid(x_t) / sum_j sigmoid(x_t)_j``) and ``c[b, e]`` the number of the ``S k``
actual selections (after bias and group limits) of sequence ``b`` that went to expert ``e``:

* ``A_b = E / (k S^2) sum_e c[b, e] sum_{t in b} s[t, e]``; 1 when balanced, up to ``E / k``.

The call's objective ``w S coef_seq sum_b A_b`` (``= w T coef_seq mean_b A_b``) is back-propagated the same way, and
``(w S sum_b A_b, w T)`` is added to an optional fp32 ``[2]`` accumulator in backward.

All of them are computed from per-sequence statistics (``c[b, e]``, ``sum_{t in b} s[t, e]``, ``sum_{t in b} lse_t^2``):
the batch losses from the rows summed, which is one sequence of all ``T`` tokens when the sequence-wise loss is off.
"""

from __future__ import annotations

from typing import Any

import torch
import torch.nn.functional as F
from torch.autograd import Function

from .._native import native_ops, on_gpu


def _balance_grad(counts: torch.Tensor, score_sum: torch.Tensor, lse2_sum: torch.Tensor, num_tokens: int, top_k: int,
                  losses: tuple) -> tuple[torch.Tensor, float]:
    """Per-sequence statistics of ``num_tokens`` tokens (``counts [B, E]``, ``score_sum [B, E] = sum_{t in b} s[t]``,
    ``lse2_sum [B] = sum_{t in b} lse_t^2``) -> the balance gradient ``g [B, E]`` fp32 (``dlogits[t] += ds_t/dx_t^T
    (g_b - s_t . g_b)``) and the z-loss factor ``2 w coef_z`` (``dlogits[t] += 2 w coef_z lse_t s_t``).  Adds
    ``(w S sum_b A_b, w T)`` to the sequence accumulator and ``(w T A, w T Z, w T)`` to the batch one; device-side, no
    host synchronisation."""
    seq_len, seq_coef, lb_coef, z_coef, token_weight, seq_sums, aux_sums = losses
    num_seqs, num_experts = counts.shape
    c = counts.float()
    g, zc = None, 0.0
    if seq_coef > 0:  # sequence-wise balance, per row: g_b = w coef E c_b / (k S)
        per_count = token_weight * num_experts / (top_k * seq_len)
        g = c * (per_count * seq_coef)
        if seq_sums is not None:
            seq_sums.add_(torch.cat([(c * score_sum.float()).sum().reshape(1) * per_count,
                                     c.new_full((1,), token_weight * num_tokens)]))
    if lb_coef > 0 or z_coef > 0:  # batch load balancing and z-loss: from the rows summed, broadcast to every row
        if num_seqs != 1:
            c, score_sum, lse2_sum = c.sum(0, keepdim=True), score_sum.sum(0, keepdim=True), lse2_sum.sum().reshape(1)
        t = max(num_tokens, 1)  # no tokens: no counts, no gradient, weight 0
        omega = token_weight * num_tokens
        g_batch = c * (token_weight * lb_coef * num_experts / (top_k * t))
        g = g_batch if g is None else g + g_batch
        zc = 2.0 * token_weight * z_coef
        if aux_sums is not None:
            aux_sums.add_(torch.cat([
                torch.dot(c.view(-1), score_sum.float().view(-1)).reshape(1) * (omega * num_experts / (top_k * t * t)),
                lse2_sum.float().reshape(1) * (omega / t),
                c.new_full((1,), omega),
            ]))
    return g, zc


def _balance_scores(x: torch.Tensor, score_function: str) -> tuple[torch.Tensor, torch.Tensor]:
    """fp32 ``x [T, E]`` -> the balance scores ``s`` and their Jacobian's diagonal factor: ``ds/dx^T v = d (v - s . v)``
    with ``d = s`` (softmax) or ``sigmoid (1 - sigmoid) / sum_j sigmoid_j`` (normalised sigmoid)."""
    if score_function == "softmax":
        s = F.softmax(x, dim=-1)
        return s, s
    sig = torch.sigmoid(x)
    total = sig.sum(-1, keepdim=True)
    return sig / total, sig * (1 - sig) / total


class _BalanceLossGrad(Function):
    """CPU path (and numerics oracle) of the auxiliary losses: identity on the selected probabilities; backward computes
    the ``num_seqs`` sequences' statistics and adds the losses' gradient to the logits' gradient, in fp32 from the plain
    PyTorch definitions."""

    @staticmethod
    def forward(ctx: Any, chosen_p: torch.Tensor, logits: torch.Tensor, chosen: torch.Tensor, top_k: int, score_function: str,
                num_seqs: int, losses: tuple):
        ctx.save_for_backward(logits.detach(), chosen)
        ctx.args = (top_k, score_function, num_seqs, losses)
        return chosen_p.view_as(chosen_p)

    @staticmethod
    def backward(ctx: Any, dprobs: torch.Tensor):  # type: ignore[override]
        logits, chosen = ctx.saved_tensors
        top_k, score_function, num_seqs, losses = ctx.args
        x = logits.reshape(-1, logits.shape[-1]).float()
        num_tokens, num_experts = x.shape
        seq_len = num_tokens // num_seqs
        s, d = _balance_scores(x, score_function)
        lse = torch.logsumexp(x, dim=-1) if score_function == "softmax" else x.new_zeros(num_tokens)
        sel = chosen.reshape(num_seqs, seq_len * top_k)
        counts = torch.zeros(num_seqs, num_experts, dtype=torch.int64, device=x.device).scatter_add_(1, sel, torch.ones_like(sel))
        g, zc = _balance_grad(counts, s.reshape(num_seqs, seq_len, num_experts).sum(1),
                              (lse * lse).reshape(num_seqs, seq_len).sum(1), num_tokens, top_k, losses)
        g = g.repeat_interleave(seq_len, dim=0)
        dlogits = d * (g - (s * g).sum(-1, keepdim=True))
        if zc:
            dlogits = dlogits + zc * lse[:, None] * s
        # autograd adds this term to the selection gradient in the logits' dtype: exact for the fp32 logits the oracle
        # is used with; for bf16 logits it is rounded once before the sum (the kernel rounds their fp32 sum)
        return dprobs, dlogits.to(logits.dtype).reshape(logits.shape), None, None, None, None, None


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
    """Routing on the fused kernel.  With auxiliary losses (``num_seqs > 0``) the same pass also produces the per-sequence
    statistics (deterministic, so a recomputed forward reproduces them bit for bit) and the losses' gradients are folded
    into the fused backward."""

    @staticmethod
    def forward(ctx: Any, logits: torch.Tensor, top_k: int, renormalize: bool, expert_bias: torch.Tensor | None,
                score_function: str, num_groups: int, topk_groups: int, scaling_factor: float, num_seqs: int,
                losses: tuple | None):
        idx, probs, counts, score_sum, lse2_sum = native_ops().router_topk_fwd(
            logits, expert_bias, top_k, renormalize, score_function, num_groups, topk_groups, scaling_factor, num_seqs)
        ctx.save_for_backward(logits, idx, counts, score_sum, lse2_sum)
        ctx.args = (renormalize, score_function, scaling_factor, top_k, losses)
        ctx.mark_non_differentiable(idx)
        return idx, probs

    @staticmethod
    def backward(ctx: Any, _didx: torch.Tensor, dprobs: torch.Tensor):  # type: ignore[override]
        logits, idx, counts, score_sum, lse2_sum = ctx.saved_tensors
        renormalize, score_function, scaling_factor, top_k, losses = ctx.args
        g, zc = (None, 0.0) if losses is None else _balance_grad(counts, score_sum, lse2_sum, logits.shape[0], top_k, losses)
        dlogits = native_ops().router_topk_bwd(logits, idx, dprobs.float().contiguous(), renormalize, score_function,
                                               scaling_factor, g, zc)
        return dlogits, *([None] * 9)


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
               score_function: str = "softmax", num_groups: int = 1, topk_groups: int = 1, scaling_factor: float = 1.0, *,
               load_balancing_coef: float = 0.0, z_loss_coef: float = 0.0, token_loss_weight: float | None = None,
               aux_loss_sums: torch.Tensor | None = None, sequence_balance_coef: float = 0.0,
               sequence_length: int | None = None, sequence_balance_sums: torch.Tensor | None = None):
    """``logits [..., E]`` -> ``(indices [..., k] int64, probabilities [..., k] fp32)``.

    bf16 CUDA logits with ``E <= 1024``, ``k <= min(32, E)`` and at most 32 expert groups run on the fused CUDA kernel,
    whatever the routing options (softmax or sigmoid scores, bias, group-limited selection, renormalisation, scaling).
    Other inputs use the PyTorch definitions: ``route_topk_reference`` for plain softmax top-k, ``route_topk_general``
    for the DeepSeek variants.

    Auxiliary losses (softmax scores only; see the module docstring): with ``load_balancing_coef > 0`` or
    ``z_loss_coef > 0`` the backward also adds the gradient of ``token_loss_weight * T * (load_balancing_coef * A +
    z_loss_coef * Z)`` to the logits, and adds ``(w T A, w T Z, w T)`` to ``aux_loss_sums`` (fp32 ``[3]``, optional).
    With both coefficients 0 the call is exactly the one without them.

    Sequence-wise balance loss (softmax or sigmoid scores; see the module docstring): with ``sequence_balance_coef > 0``
    the tokens are ``T / sequence_length`` sequences of ``sequence_length`` consecutive tokens (it must divide ``T``), the
    backward also adds the gradient of ``token_loss_weight * sequence_length * sequence_balance_coef * sum_b A_b`` and adds
    ``(w S sum_b A_b, w T)`` to ``sequence_balance_sums`` (fp32 ``[2]``, optional).  With the coefficient 0 the call is
    exactly the one without it.
    """
    num_experts = logits.shape[-1]
    if num_groups > 1 and (num_experts % num_groups != 0 or not 0 < topk_groups <= num_groups):
        raise ValueError("experts must split evenly into groups and 0 < topk_groups <= num_groups")
    if score_function not in ("softmax", "sigmoid"):
        raise ValueError(f"unknown router score function {score_function!r}")
    if load_balancing_coef < 0 or z_loss_coef < 0:
        raise ValueError("auxiliary loss coefficients must be non-negative")
    aux = load_balancing_coef > 0 or z_loss_coef > 0
    if aux:
        if score_function != "softmax":
            raise ValueError("the load-balancing and z auxiliary losses are defined for softmax routers only")
        if token_loss_weight is None:
            raise ValueError("auxiliary losses need token_loss_weight, the loss weight of one token")
        if aux_loss_sums is not None and (aux_loss_sums.dtype != torch.float32 or aux_loss_sums.shape != (3,)
                                          or aux_loss_sums.device != logits.device):
            raise ValueError("aux_loss_sums must be an fp32 [3] tensor on the logits' device")
    if sequence_balance_coef < 0:
        raise ValueError("the sequence balance coefficient must be non-negative")
    seq = sequence_balance_coef > 0
    if seq:
        if token_loss_weight is None:
            raise ValueError("auxiliary losses need token_loss_weight, the loss weight of one token")
        num_tokens = logits.shape[:-1].numel()
        if sequence_length is None or sequence_length < 1 or num_tokens % sequence_length != 0:
            raise ValueError(f"the sequence-wise balance loss needs sequence_length, a positive divisor of the token count "
                             f"({num_tokens}), got {sequence_length}")
        if sequence_balance_sums is not None and (sequence_balance_sums.dtype != torch.float32
                                                  or sequence_balance_sums.shape != (2,)
                                                  or sequence_balance_sums.device != logits.device):
            raise ValueError("sequence_balance_sums must be an fp32 [2] tensor on the logits' device")
    # statistics per sequence: T / S sequences for the sequence-wise loss (one empty one without tokens), one for the batch
    # losses alone, none without a loss
    num_seqs = max(logits.shape[:-1].numel() // sequence_length, 1) if seq else int(aux)
    losses = None
    if aux or seq:
        losses = (sequence_length, float(sequence_balance_coef), float(load_balancing_coef), float(z_loss_coef),
                  float(token_loss_weight), sequence_balance_sums, aux_loss_sums)
    if (on_gpu(logits) and logits.dtype == torch.bfloat16 and num_experts <= 1024 and top_k <= min(32, num_experts)
            and num_groups <= 32):
        flat = logits.reshape(logits.shape[:-1].numel(), num_experts)  # also when there are no tokens
        if not flat.is_contiguous():
            flat = flat.contiguous()
        groups = (num_groups, topk_groups) if num_groups > 1 else (1, 1)
        bias = None if expert_bias is None else expert_bias.float().contiguous()
        idx, probs = _RouteTopK.apply(flat, top_k, renormalize, bias, score_function, *groups, float(scaling_factor),
                                      num_seqs, losses)
        return idx.view(*logits.shape[:-1], top_k), probs.view(*logits.shape[:-1], top_k)
    if score_function != "softmax" or num_groups > 1 or scaling_factor != 1.0:
        chosen, chosen_p = route_topk_general(logits, top_k, renormalize, expert_bias, score_function, num_groups, topk_groups,
                                              scaling_factor)
    else:
        chosen, chosen_p = route_topk_reference(logits, top_k, renormalize, expert_bias)
    if losses is not None:
        chosen_p = _BalanceLossGrad.apply(chosen_p, logits, chosen, top_k, score_function, num_seqs, losses)
    return chosen, chosen_p


__all__ = ["route_topk", "route_topk_general", "route_topk_reference"]
