from __future__ import annotations

import torch
from torch import nn

from d9d_b200.kernel.gemm import linear


class Linear(nn.Linear):
    """``nn.Linear`` (same parameters / state-dict keys / init) whose matmuls run on the hand-written wgmma GEMM."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:  # noqa: D102
        return linear(x, self.weight, self.bias)
