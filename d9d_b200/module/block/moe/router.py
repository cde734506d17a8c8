from __future__ import annotations

import dataclasses
from typing import Literal

import torch
from pydantic import BaseModel, PositiveInt
from torch import nn

from d9d_b200.kernel.router import route_topk
from d9d_b200.module.base import ModuleLateInit
from d9d_b200.module.block.linear import Linear


@dataclasses.dataclass(kw_only=True, slots=True)
class RoutingResult:
    selected_expert_indices: torch.Tensor  # [T, k] int64
    selected_probabilities: torch.Tensor  # [T, k] fp32


class RouterParameters(BaseModel):
    """Routing variants beyond the plain softmax top-k (DeepSeek-V2 / V3)."""

    score_function: Literal["softmax", "sigmoid"] = "softmax"
    enable_expert_bias: bool = False  # selection bias buffer for auxiliary-loss-free load balancing
    num_expert_groups: PositiveInt = 1  # group-limited routing: experts are split into this many groups ...
    topk_expert_groups: PositiveInt = 1  # ... of which only the best ones stay eligible
    routed_scaling_factor: float = 1.0


class TopKRouter(nn.Module, ModuleLateInit):
    """Linear gate -> fp32 softmax over all experts -> top-k (optionally biased selection) -> optional renorm
    (softmax / selection / renormalisation are one fused kernel on CUDA, ``ops/csrc/router.cu``).

    Softmax routers can also train with the load-balancing and router z auxiliary losses (``set_aux_loss``, off by
    default; definitions in ``d9d_b200.kernel.router``): their gradients are added in the router's backward, and
    ``aux_loss_sums`` (fp32, not saved) accumulates ``(sum w T A, sum w T Z, sum w T)`` over the backward passes since
    ``reset_aux_loss_sums``.  Softmax and sigmoid routers can train with the sequence-wise balance loss
    (``set_sequence_balance_loss``, off by default): ``forward`` then needs the sequence length, and
    ``sequence_balance_sums`` (fp32, not saved) accumulates ``(sum w S sum_b A_b, sum w T)``.

    Parity: reference ``d9d/module/block/moe/router.py:24-107``.
    """

    def __init__(self, dim: int, num_experts: int, top_k: int, renormalize_probabilities: bool,
                 enable_expert_bias: bool = False, options: RouterParameters | None = None) -> None:
        super().__init__()
        options = options if options is not None else RouterParameters(enable_expert_bias=enable_expert_bias)
        self.gate = Linear(dim, num_experts, bias=False)
        self.expert_bias: nn.Buffer | None = (
            nn.Buffer(torch.empty(num_experts, dtype=torch.float32), persistent=True)
            if (enable_expert_bias or options.enable_expert_bias) else None
        )
        self.aux_loss_sums = nn.Buffer(torch.empty(3, dtype=torch.float32), persistent=False)
        self.sequence_balance_sums = nn.Buffer(torch.empty(2, dtype=torch.float32), persistent=False)
        self._num_experts = num_experts
        self._top_k = top_k
        self._renormalize = renormalize_probabilities
        self._options = options
        self._load_balancing_coef = 0.0
        self._z_loss_coef = 0.0
        self._token_loss_weight: float | None = None
        self._sequence_balance_coef = 0.0

    @property
    def score_function(self) -> str:
        return self._options.score_function

    def set_aux_loss(self, load_balancing_coef: float, z_loss_coef: float, token_loss_weight: float) -> None:
        """Train with ``token_loss_weight * T * (load_balancing_coef * A + z_loss_coef * Z)`` per forward of ``T``
        tokens (softmax routers only; both coefficients 0 switch the losses off)."""
        if load_balancing_coef < 0 or z_loss_coef < 0:
            raise ValueError("auxiliary loss coefficients must be non-negative")
        if (load_balancing_coef > 0 or z_loss_coef > 0) and self.score_function != "softmax":
            raise ValueError(f"the load-balancing and z auxiliary losses need a softmax router, not {self.score_function!r} "
                             "(sigmoid routers balance with the expert bias)")
        self._load_balancing_coef = float(load_balancing_coef)
        self._z_loss_coef = float(z_loss_coef)
        self._token_loss_weight = float(token_loss_weight)

    @property
    def sequence_balance_coef(self) -> float:
        return self._sequence_balance_coef

    def set_sequence_balance_loss(self, coef: float, token_loss_weight: float) -> None:
        """Train with ``token_loss_weight * S * coef * sum_b A_b`` per forward of sequences of ``S`` tokens (softmax or
        sigmoid routers; coefficient 0 switches the loss off)."""
        if coef < 0:
            raise ValueError("the sequence balance coefficient must be non-negative")
        self._sequence_balance_coef = float(coef)
        self._token_loss_weight = float(token_loss_weight)

    @torch.no_grad()
    def reset_aux_loss_sums(self) -> None:
        """Zero ``aux_loss_sums`` and ``sequence_balance_sums``."""
        for name, size in (("aux_loss_sums", 3), ("sequence_balance_sums", 2)):
            sums = getattr(self, name)
            if sums.dtype == torch.float32:
                sums.zero_()
            else:  # the module was cast whole: the sums stay fp32
                setattr(self, name, torch.zeros(size, dtype=torch.float32, device=sums.device))

    def forward(self, hidden_states: torch.Tensor, sequence_length: int | None = None) -> RoutingResult:
        """``hidden_states [T, D]``; ``sequence_length``: tokens per sequence (the sequence-wise balance loss needs it)."""
        o = self._options
        aux = {}
        if self._load_balancing_coef > 0 or self._z_loss_coef > 0:
            aux = {"load_balancing_coef": self._load_balancing_coef, "z_loss_coef": self._z_loss_coef,
                   "token_loss_weight": self._token_loss_weight, "aux_loss_sums": self.aux_loss_sums}
        if self._sequence_balance_coef > 0:
            aux |= {"sequence_balance_coef": self._sequence_balance_coef, "sequence_length": sequence_length,
                    "token_loss_weight": self._token_loss_weight, "sequence_balance_sums": self.sequence_balance_sums}
        chosen, chosen_p = route_topk(self.gate(hidden_states), self._top_k, self._renormalize, self.expert_bias,
                                      score_function=o.score_function, num_groups=o.num_expert_groups,
                                      topk_groups=o.topk_expert_groups, scaling_factor=o.routed_scaling_factor, **aux)
        return RoutingResult(selected_expert_indices=chosen, selected_probabilities=chosen_p)

    def reset_parameters(self) -> None:
        if self.expert_bias is not None:
            nn.init.zeros_(self.expert_bias)
        self.gate.reset_parameters()
        self.reset_aux_loss_sums()
