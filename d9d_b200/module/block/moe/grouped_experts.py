from __future__ import annotations

import torch
from torch import nn

from torch.distributed.tensor import DTensor

from d9d_b200.kernel._native import MAIN_PARAM_ATTR
from d9d_b200.kernel.moe import MoELayout, grouped_swiglu
from d9d_b200.kernel.swiglu import silu_mul, silu_mul_probs
from d9d_b200.module.base import ModuleLateInit

from .grouped_linear import GroupedLinear


def _local_weight(linear: GroupedLinear) -> torch.Tensor:
    weight: torch.Tensor = linear.weight
    if isinstance(weight, DTensor):
        local = weight.to_local()
        setattr(local, MAIN_PARAM_ATTR, linear.weight)  # wgrad accumulates straight into the sharded .grad
        return local
    return weight


class GroupedSwiGLU(nn.Module, ModuleLateInit):
    """All experts' SwiGLU FFNs as three grouped GEMMs: ``probs * down(silu(gate(x)) * up(x))``.

    Parity: reference ``d9d/module/block/moe/grouped_experts.py:10-73``.  On the native path the routing probability
    is folded into the SiLU·mul kernel (``down`` is linear, so scaling its input equals scaling its output).
    """

    def __init__(self, hidden_dim: int, intermediate_dim: int, num_experts: int):
        super().__init__()
        self._num_experts = num_experts
        self.gate_proj = GroupedLinear(num_experts, hidden_dim, intermediate_dim)
        self.up_proj = GroupedLinear(num_experts, hidden_dim, intermediate_dim)
        self.down_proj = GroupedLinear(num_experts, intermediate_dim, hidden_dim)

    def forward(self, permuted_x: torch.Tensor, permuted_probs: torch.Tensor,
                tokens_per_expert: torch.Tensor | MoELayout, out: torch.Tensor | None = None,
                dx_out: torch.Tensor | None = None) -> torch.Tensor:
        """``out`` / ``dx_out`` (optional, fused CUDA path only): buffers the block writes its output / its input gradient
        into - the expert-parallel handler passes its NVLink staging region so that the peers read them in place."""
        if permuted_x.numel() == 0:
            return permuted_x
        if (isinstance(tokens_per_expert, MoELayout) and permuted_x.is_cuda and permuted_x.dtype == torch.bfloat16
                and all(type(m) is GroupedLinear for m in (self.gate_proj, self.up_proj, self.down_proj))):
            # one autograd node for the whole block (plain projections only: adapters such as LoRA compose the slow way)
            return grouped_swiglu(permuted_x, permuted_probs, _local_weight(self.gate_proj), _local_weight(self.up_proj),
                                  _local_weight(self.down_proj), tokens_per_expert, out, dx_out)
        gate = self.gate_proj(permuted_x, tokens_per_expert)
        up = self.up_proj(permuted_x, tokens_per_expert)
        if isinstance(tokens_per_expert, MoELayout):
            return self.down_proj(silu_mul_probs(gate, up, permuted_probs), tokens_per_expert)
        out = self.down_proj(silu_mul(gate, up), tokens_per_expert)
        return permuted_probs[:, None].to(out.dtype) * out

    def reset_parameters(self) -> None:
        self.gate_proj.reset_parameters()
        self.up_proj.reset_parameters()
        self.down_proj.reset_parameters()
