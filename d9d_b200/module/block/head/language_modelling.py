from __future__ import annotations

from collections.abc import Sequence

import torch
from torch import nn

from d9d_b200.kernel.cce import linear_cross_entropy
from d9d_b200.module.base import ModuleLateInit

LM_IGNORE_INDEX = -100
"""Label value skipped by the LM head (loss 0 at that position)."""


class SplitLanguageModellingHead(nn.Module, ModuleLateInit):
    """LM head stored as named vocabulary splits; returns the *per-token* loss without materialising logits: the NLL, or
    the regularised training objective once ``set_loss_regularisation`` was called.

    Parity: reference ``d9d/module/block/head/language_modelling.py:10-76`` (keys ``lm_head.{split}.weight``).
    """

    def __init__(self, split_vocab_size: dict[str, int], split_order: Sequence[str], hidden_size: int):
        super().__init__()
        self.lm_head = nn.ModuleDict({name: nn.Linear(hidden_size, size, bias=False) for name, size in split_vocab_size.items()})
        self._split_order = tuple(split_order)
        self._hidden_size = hidden_size
        # (sum nll, sum lse^2, count) over the non-ignored tokens of the backward passes since reset_loss_sums
        self.lm_loss_sums = nn.Buffer(torch.zeros(3, dtype=torch.float32), persistent=False)
        self._regularisation: tuple[float, float] | None = None

    def set_loss_regularisation(self, label_smoothing: float, z_loss_coef: float) -> None:
        """Train with ``cross_entropy(z, y, label_smoothing) + z_loss_coef * lse^2`` per token and accumulate the plain
        NLL and ``lse^2`` into ``lm_loss_sums`` (both coefficients 0: the NLL, still accumulated)."""
        if not (0.0 <= label_smoothing <= 1.0) or not (0.0 <= z_loss_coef < float("inf")):
            raise ValueError(f"label_smoothing must lie in [0, 1] and z_loss_coef be finite and >= 0, got "
                             f"{label_smoothing}, {z_loss_coef}")
        self._regularisation = (float(label_smoothing), float(z_loss_coef))

    @torch.no_grad()
    def reset_loss_sums(self) -> None:
        if self.lm_loss_sums.dtype == torch.float32:
            self.lm_loss_sums.zero_()
        else:  # the module was cast whole: the sums stay fp32
            self.lm_loss_sums = torch.zeros(3, dtype=torch.float32, device=self.lm_loss_sums.device)

    def classifier_weight(self) -> torch.Tensor:
        parts = [self.lm_head[name].weight for name in self._split_order]
        return parts[0] if len(parts) == 1 else torch.cat(parts, dim=0)

    def classifier_blocks(self) -> list[torch.Tensor]:
        """The classifier as row blocks in vocabulary order (consumed in place by the fused linear-CE kernels)."""
        return [self.lm_head[name].weight for name in self._split_order]

    def forward(self, hidden_states: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        if self._regularisation is None:
            return linear_cross_entropy(hidden_states, self.classifier_blocks(), labels, ignore_index=LM_IGNORE_INDEX,
                                        reduction="none")
        label_smoothing, z_loss_coef = self._regularisation
        return linear_cross_entropy(hidden_states, self.classifier_blocks(), labels, ignore_index=LM_IGNORE_INDEX,
                                    reduction="none", label_smoothing=label_smoothing, z_loss_coef=z_loss_coef,
                                    loss_sums=self.lm_loss_sums)

    def reset_parameters(self) -> None:
        for head in self.lm_head.values():
            head.reset_parameters()
        self.reset_loss_sums()
