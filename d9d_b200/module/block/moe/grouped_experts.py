from __future__ import annotations

import torch
from torch import nn

from torch.distributed.tensor import DTensor

from d9d_b200.kernel._native import MAIN_PARAM_ATTR
from d9d_b200.kernel.moe import MoELayout, grouped_swiglu, grouped_swiglu_fp8_reference
from d9d_b200.kernel.moe.experts import FP8_EXPERT_RECIPES
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
        self.fp8 = False
        self.fp8_recipe = "rowwise"
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
        plain = self._plain_projections()
        if (isinstance(tokens_per_expert, MoELayout) and permuted_x.is_cuda and permuted_x.dtype == torch.bfloat16
                and plain):
            # one autograd node for the whole block (plain projections only: adapters such as LoRA compose the slow way)
            return grouped_swiglu(permuted_x, permuted_probs, _local_weight(self.gate_proj), _local_weight(self.up_proj),
                                  _local_weight(self.down_proj), tokens_per_expert, out, dx_out, fp8=self.fp8,
                                  recipe=self.fp8_recipe)
        if self.fp8:
            return self._fp8_emulation(permuted_x, permuted_probs, tokens_per_expert, plain)
        gate = self.gate_proj(permuted_x, tokens_per_expert)
        up = self.up_proj(permuted_x, tokens_per_expert)
        if isinstance(tokens_per_expert, MoELayout):
            return self.down_proj(silu_mul_probs(gate, up, permuted_probs), tokens_per_expert)
        out = self.down_proj(silu_mul(gate, up), tokens_per_expert)
        return permuted_probs[:, None].to(out.dtype) * out

    def _plain_projections(self) -> bool:
        return all(type(m) is GroupedLinear for m in (self.gate_proj, self.up_proj, self.down_proj))

    def enable_fp8(self, recipe: str = "rowwise") -> None:
        """Run the six expert GEMMs in e4m3 (``grouped_swiglu(..., fp8=True, recipe=recipe)``); the weights stay bf16.
        ``recipe="rowwise"`` uses per-expert row / column scales, ``"blockwise"`` DeepSeek-V3's 1x128 activation / 128x128
        weight scales with per-k-block promotion.  Hidden and intermediate sizes must be multiples of 16; LoRA-wrapped
        projections and unknown recipes are refused.

        On CUDA only the fused path runs (bf16 activations in a :class:`MoELayout`, which :class:`MoELayer` always
        passes); a per-expert counts tensor or other activation dtypes are refused there rather than emulated.  On CPU
        the block runs the PyTorch emulation of the recipe (``grouped_swiglu_fp8_reference``) for either grouping."""
        if recipe not in FP8_EXPERT_RECIPES:
            raise ValueError(f"GroupedSwiGLU.enable_fp8: unknown recipe {recipe!r} (expected one of {FP8_EXPERT_RECIPES})")
        if not self._plain_projections():
            raise ValueError("GroupedSwiGLU.enable_fp8: the expert projections are wrapped (LoRA or another adapter); fp8 "
                             "experts need plain GroupedLinear projections")
        sizes = (self.gate_proj.in_features, self.gate_proj.out_features)
        if any(d % 16 for d in sizes):
            raise ValueError(f"GroupedSwiGLU.enable_fp8: hidden and intermediate sizes must be multiples of 16, got {sizes}")
        self.fp8 = True
        self.fp8_recipe = recipe

    def _fp8_emulation(self, x: torch.Tensor, probs: torch.Tensor, groups: torch.Tensor | MoELayout, plain: bool) -> torch.Tensor:
        """The fp8 recipe in PyTorch, for CPU tensors (the CUDA path has no emulation: it runs the native kernels only)."""
        if not plain:
            raise ValueError("GroupedSwiGLU: fp8 experts need plain GroupedLinear projections (LoRA is not supported)")
        if x.is_cuda:
            raise RuntimeError("GroupedSwiGLU: fp8 experts on CUDA need bf16 activations in the MoE layout (MoELayout)")
        if isinstance(groups, MoELayout):
            starts, counts = groups.seg_offsets[:-1].tolist(), groups.counts.tolist()
        else:
            counts = [int(c) for c in groups.tolist()]
            starts = [sum(counts[:e]) for e in range(len(counts))]
        return grouped_swiglu_fp8_reference(x, probs, _local_weight(self.gate_proj), _local_weight(self.up_proj),
                                            _local_weight(self.down_proj), starts, counts, self.fp8_recipe)

    def reset_parameters(self) -> None:
        self.gate_proj.reset_parameters()
        self.up_proj.reset_parameters()
        self.down_proj.reset_parameters()
