from __future__ import annotations

import math

import torch
from torch import nn
from torch.distributed.tensor import DTensor

from d9d_b200.core.autograd import GradDirection
from d9d_b200.kernel._native import MAIN_PARAM_ATTR
from d9d_b200.kernel.gmm import gmm
from d9d_b200.kernel.moe import MoELayout, grouped_linear
from d9d_b200.module.base import ModuleLateInit


class GroupedLinear(nn.Module, ModuleLateInit):
    """``E`` independent linear maps with weight ``[E, in, out]`` applied to expert-sorted rows.

    ``x_groups`` is either a device-side :class:`MoELayout` (native path: aligned layout, wgmma grouped GEMM, no host
    sync) or — for compatibility with the reference contract (``d9d/module/block/moe/grouped_linear.py:12-71``) —
    a CPU tensor with the number of rows per expert.
    """

    def __init__(self, n_groups: int, in_features: int, out_features: int, device: torch.device | str | None = None,
                 dtype: torch.dtype | None = None):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(n_groups, in_features, out_features, device=device, dtype=dtype))
        self.n_groups = n_groups
        self.in_features = in_features
        self.out_features = out_features
        self.reset_parameters()

    def forward(self, x: torch.Tensor, x_groups: torch.Tensor | MoELayout) -> torch.Tensor:
        weight: torch.Tensor = self.weight
        if isinstance(weight, DTensor):
            weight = weight.to_local()
            setattr(weight, MAIN_PARAM_ATTR, self.weight)  # wgrad accumulates straight into the sharded .grad
        if isinstance(x_groups, MoELayout):
            return grouped_linear(x, weight, x_groups)
        return gmm(x, weight, x_groups, a_grad_direction=GradDirection.inputs, b_grad_direction=GradDirection.weight)

    def reset_parameters(self) -> None:
        if self.weight.is_meta:
            return
        bound = 1.0 / math.sqrt(self.in_features)
        nn.init.uniform_(self.weight, -bound, bound)

    def extra_repr(self) -> str:
        return f"groups={self.n_groups}, in={self.in_features}, out={self.out_features}"
