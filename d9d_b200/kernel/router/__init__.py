"""Fused MoE routing: fp32 softmax or sigmoid scores + top-k (+ selection bias, + group-limited selection, + renormalisation,
+ scaling) and its backward, optionally with the softmax router's auxiliary losses folded into that backward.

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
"""

from __future__ import annotations

from typing import Any

import torch
import torch.nn.functional as F
from torch.autograd import Function

from .._native import native_ops, on_gpu


def _aux_terms(counts: torch.Tensor, score_sum: torch.Tensor, lse2_sum: torch.Tensor, num_tokens: int, top_k: int,
               lb_coef: float, z_coef: float, token_weight: float) -> tuple[torch.Tensor, float, torch.Tensor]:
    """One call's statistics (``counts [E]``, ``score_sum [E] = sum_t s[t]``, ``lse2_sum [1] = sum_t lse_t^2``) ->
    ``g [E]`` fp32 (load balancing: ``dlogits[t] += s_t (g - s_t . g)``), the z-loss factor ``2 w coef_z``
    (``dlogits[t] += 2 w coef_z lse_t s_t``) and ``(w T A, w T Z, w T)`` fp32 ``[3]``."""
    num_experts = counts.numel()
    t = max(num_tokens, 1)  # no tokens: no counts, no gradient, weight 0
    omega = token_weight * num_tokens
    c = counts.float()
    g = c * (token_weight * lb_coef * num_experts / (top_k * t))
    logged = torch.cat([
        torch.dot(c, score_sum.float()).reshape(1) * (omega * num_experts / (top_k * t * t)),
        lse2_sum.float().reshape(1) * (omega / t),
        lse2_sum.new_full((1,), omega, dtype=torch.float32),
    ])
    return g, 2.0 * token_weight * z_coef, logged


class _AuxLossGrad(Function):
    """CPU path (and numerics oracle) of the auxiliary losses: identity on the selected probabilities; backward adds
    ``w T (coef_lb grad A + coef_z grad Z)`` to the logits' gradient, in fp32 from the plain PyTorch definitions."""

    @staticmethod
    def forward(ctx: Any, chosen_p: torch.Tensor, logits: torch.Tensor, chosen: torch.Tensor, top_k: int, lb_coef: float,
                z_coef: float, token_weight: float, sums: torch.Tensor | None):
        ctx.save_for_backward(logits.detach(), chosen)
        ctx.args = (top_k, lb_coef, z_coef, token_weight, sums)
        return chosen_p.view_as(chosen_p)

    @staticmethod
    def backward(ctx: Any, dprobs: torch.Tensor):  # type: ignore[override]
        logits, chosen = ctx.saved_tensors
        top_k, lb_coef, z_coef, token_weight, sums = ctx.args
        x = logits.reshape(-1, logits.shape[-1]).float()
        s = F.softmax(x, dim=-1)
        lse = torch.logsumexp(x, dim=-1)
        counts = torch.bincount(chosen.reshape(-1), minlength=x.shape[-1])
        g, zc, logged = _aux_terms(counts, s.sum(0), (lse * lse).sum().reshape(1), x.shape[0], top_k, lb_coef, z_coef,
                                   token_weight)
        dlogits = s * (g - (s @ g)[:, None]) + zc * lse[:, None] * s
        if sums is not None:
            sums.add_(logged)
        # autograd adds this term to the selection gradient in the logits' dtype: exact for the fp32 logits the oracle
        # is used with; for bf16 logits each term is rounded once before the sum (the kernel rounds their fp32 sum)
        return dprobs, dlogits.to(logits.dtype).reshape(logits.shape), None, None, None, None, None, None


def _seq_balance_terms(counts: torch.Tensor, score_sum: torch.Tensor, seq_len: int, top_k: int, coef: float,
                       token_weight: float) -> tuple[torch.Tensor, torch.Tensor]:
    """Per-sequence statistics (``counts [B, E]``, ``score_sum [B, E] = sum_{t in b} s[t]``) -> ``g [B, E]`` fp32
    (``dlogits[t] += ds_t/dx_t^T (g_b - s_t . g_b)``, ``g_b = w coef E c_b / (k S)``) and ``(w S sum_b A_b, w T)``
    fp32 ``[2]``; device-side, no host synchronisation."""
    num_seqs, num_experts = counts.shape
    c = counts.float()
    per_count = token_weight * num_experts / (top_k * seq_len)
    logged = torch.cat([(c * score_sum.float()).sum().reshape(1) * per_count,
                        counts.new_full((1,), token_weight * num_seqs * seq_len, dtype=torch.float32)])
    return c * (per_count * coef), logged


def _balance_scores(x: torch.Tensor, score_function: str) -> tuple[torch.Tensor, torch.Tensor]:
    """fp32 ``x [T, E]`` -> the balance scores ``s`` and their Jacobian's diagonal factor: ``ds/dx^T v = d (v - s . v)``
    with ``d = s`` (softmax) or ``sigmoid (1 - sigmoid) / sum_j sigmoid_j`` (normalised sigmoid)."""
    if score_function == "softmax":
        s = F.softmax(x, dim=-1)
        return s, s
    sig = torch.sigmoid(x)
    total = sig.sum(-1, keepdim=True)
    return sig / total, sig * (1 - sig) / total


class _SeqBalanceGrad(Function):
    """CPU path (and numerics oracle) of the sequence-wise balance loss: identity on the selected probabilities; backward
    adds ``w S coef_seq grad sum_b A_b`` to the logits' gradient, in fp32 from the plain PyTorch definition."""

    @staticmethod
    def forward(ctx: Any, chosen_p: torch.Tensor, logits: torch.Tensor, chosen: torch.Tensor, top_k: int, score_function: str,
                seq_len: int, coef: float, token_weight: float, sums: torch.Tensor | None):
        ctx.save_for_backward(logits.detach(), chosen)
        ctx.args = (top_k, score_function, seq_len, coef, token_weight, sums)
        return chosen_p.view_as(chosen_p)

    @staticmethod
    def backward(ctx: Any, dprobs: torch.Tensor):  # type: ignore[override]
        logits, chosen = ctx.saved_tensors
        top_k, score_function, seq_len, coef, token_weight, sums = ctx.args
        x = logits.reshape(-1, logits.shape[-1]).float()
        num_seqs, num_experts = x.shape[0] // seq_len, x.shape[1]
        s, d = _balance_scores(x, score_function)
        sel = chosen.reshape(num_seqs, seq_len * top_k)
        counts = torch.zeros(num_seqs, num_experts, dtype=torch.int64, device=x.device).scatter_add_(1, sel, torch.ones_like(sel))
        g, logged = _seq_balance_terms(counts, s.reshape(num_seqs, seq_len, num_experts).sum(1), seq_len, top_k, coef,
                                       token_weight)
        g = g.repeat_interleave(seq_len, dim=0)
        dlogits = d * (g - (s * g).sum(-1, keepdim=True))
        if sums is not None:
            sums.add_(logged)
        return dprobs, dlogits.to(logits.dtype).reshape(logits.shape), None, None, None, None, None, None, None


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


class _RouteTopKAux(Function):
    """Softmax routing on the fused kernel with the auxiliary-loss statistics from the same pass (deterministic, so a
    recomputed forward reproduces them bit for bit) and both auxiliary gradients folded into the fused backward."""

    @staticmethod
    def forward(ctx: Any, logits: torch.Tensor, top_k: int, renormalize: bool, expert_bias: torch.Tensor | None,
                num_groups: int, topk_groups: int, scaling_factor: float, lb_coef: float, z_coef: float, token_weight: float,
                sums: torch.Tensor | None):
        idx, probs, counts, score_sum, lse2_sum = native_ops().router_topk_aux_fwd(
            logits, expert_bias, top_k, renormalize, num_groups, topk_groups, scaling_factor)
        ctx.save_for_backward(logits, idx, counts, score_sum, lse2_sum)
        ctx.args = (renormalize, scaling_factor, top_k, lb_coef, z_coef, token_weight, sums)
        ctx.mark_non_differentiable(idx)
        return idx, probs

    @staticmethod
    def backward(ctx: Any, _didx: torch.Tensor, dprobs: torch.Tensor):  # type: ignore[override]
        logits, idx, counts, score_sum, lse2_sum = ctx.saved_tensors
        renormalize, scaling_factor, top_k, lb_coef, z_coef, token_weight, sums = ctx.args
        g, zc, logged = _aux_terms(counts, score_sum, lse2_sum, logits.shape[0], top_k, lb_coef, z_coef, token_weight)
        dlogits = native_ops().router_topk_aux_bwd(logits, idx, dprobs.float().contiguous(), renormalize, scaling_factor, g, zc)
        if sums is not None:
            sums.add_(logged)
        return dlogits, None, None, None, None, None, None, None, None, None, None


class _RouteTopKSeq(Function):
    """Routing on the fused kernel with per-sequence statistics from the same pass (deterministic, so a recomputed forward
    reproduces them bit for bit) and the sequence-wise balance gradient - plus, for softmax, the batch load-balancing and
    z-loss gradients, whose statistics are the per-sequence ones summed - folded into the fused backward."""

    @staticmethod
    def forward(ctx: Any, logits: torch.Tensor, top_k: int, renormalize: bool, expert_bias: torch.Tensor | None,
                score_function: str, num_groups: int, topk_groups: int, scaling_factor: float, seq_len: int, seq_coef: float,
                lb_coef: float, z_coef: float, token_weight: float, seq_sums: torch.Tensor | None,
                aux_sums: torch.Tensor | None):
        idx, probs, counts, score_sum, lse2_sum = native_ops().router_topk_seq_fwd(
            logits, expert_bias, top_k, renormalize, score_function, num_groups, topk_groups, scaling_factor, seq_len)
        ctx.save_for_backward(logits, idx, counts, score_sum, lse2_sum)
        ctx.args = (renormalize, score_function, scaling_factor, top_k, seq_len, seq_coef, lb_coef, z_coef, token_weight,
                    seq_sums, aux_sums)
        ctx.mark_non_differentiable(idx)
        return idx, probs

    @staticmethod
    def backward(ctx: Any, _didx: torch.Tensor, dprobs: torch.Tensor):  # type: ignore[override]
        logits, idx, counts, score_sum, lse2_sum = ctx.saved_tensors
        (renormalize, score_function, scaling_factor, top_k, seq_len, seq_coef, lb_coef, z_coef, token_weight, seq_sums,
         aux_sums) = ctx.args
        g, logged = _seq_balance_terms(counts, score_sum, seq_len, top_k, seq_coef, token_weight)
        zc = 0.0
        if lb_coef > 0 or z_coef > 0:
            g_batch, zc, aux_logged = _aux_terms(counts.sum(0), score_sum.sum(0), lse2_sum.sum().reshape(1), logits.shape[0],
                                                 top_k, lb_coef, z_coef, token_weight)
            g = g + g_batch
            if aux_sums is not None:
                aux_sums.add_(aux_logged)
        dlogits = native_ops().router_topk_seq_bwd(logits, idx, dprobs.float().contiguous(), renormalize, score_function,
                                                   scaling_factor, g.contiguous(), zc, seq_len)
        if seq_sums is not None:
            seq_sums.add_(logged)
        return dlogits, *([None] * 14)


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
    if (on_gpu(logits) and logits.dtype == torch.bfloat16 and num_experts <= 1024 and top_k <= min(32, num_experts)
            and num_groups <= 32):
        flat = logits.reshape(logits.shape[:-1].numel(), num_experts)  # also when there are no tokens
        if not flat.is_contiguous():
            flat = flat.contiguous()
        groups = (num_groups, topk_groups) if num_groups > 1 else (1, 1)
        bias = None if expert_bias is None else expert_bias.float().contiguous()
        if seq:
            idx, probs = _RouteTopKSeq.apply(flat, top_k, renormalize, bias, score_function, *groups, float(scaling_factor),
                                             int(sequence_length), float(sequence_balance_coef), float(load_balancing_coef),
                                             float(z_loss_coef), float(token_loss_weight), sequence_balance_sums,
                                             aux_loss_sums)
        elif aux:
            idx, probs = _RouteTopKAux.apply(flat, top_k, renormalize, bias, *groups, float(scaling_factor),
                                             float(load_balancing_coef), float(z_loss_coef), float(token_loss_weight),
                                             aux_loss_sums)
        else:
            idx, probs = _RouteTopK.apply(flat, top_k, renormalize, bias, score_function, *groups, float(scaling_factor))
        return idx.view(*logits.shape[:-1], top_k), probs.view(*logits.shape[:-1], top_k)
    if score_function != "softmax" or num_groups > 1 or scaling_factor != 1.0:
        chosen, chosen_p = route_topk_general(logits, top_k, renormalize, expert_bias, score_function, num_groups, topk_groups,
                                              scaling_factor)
    else:
        chosen, chosen_p = route_topk_reference(logits, top_k, renormalize, expert_bias)
    if aux:
        chosen_p = _AuxLossGrad.apply(chosen_p, logits, chosen, top_k, float(load_balancing_coef), float(z_loss_coef),
                                      float(token_loss_weight), aux_loss_sums)
    if seq:
        chosen_p = _SeqBalanceGrad.apply(chosen_p, logits, chosen, top_k, score_function, int(sequence_length),
                                         float(sequence_balance_coef), float(token_loss_weight), sequence_balance_sums)
    return chosen, chosen_p


__all__ = ["route_topk", "route_topk_general", "route_topk_reference"]
