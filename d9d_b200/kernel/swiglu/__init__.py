"""SiLU(x)*y (reference ``d9d/kernel/swiglu/op.py``). Also the MoE variant fused with the routing probability."""

from __future__ import annotations

from typing import Any

import torch
from torch.autograd import Function

from .._native import contiguous_aligned, native_ops, on_gpu


def silu_mul_reference(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    return (torch.nn.functional.silu(x.float()).to(y.dtype).float() * y.float()).to(x.dtype)


class SiLUMulFunction(Function):
    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        x, y = contiguous_aligned(x), contiguous_aligned(y)
        ctx.save_for_backward(x, y)
        return native_ops().silu_mul_fwd(x, y)

    @staticmethod
    def backward(ctx: Any, grad_output: torch.Tensor):  # type: ignore[override]
        x, y = ctx.saved_tensors
        return native_ops().silu_mul_bwd(contiguous_aligned(grad_output), x, y)


def silu_mul(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    if on_gpu(x):
        return SiLUMulFunction.apply(x, y)
    return silu_mul_reference(x, y)


class SiLUMulProbsFunction(Function):
    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, y: torch.Tensor, probs: torch.Tensor) -> torch.Tensor:
        x, y, probs = contiguous_aligned(x), contiguous_aligned(y), probs.contiguous()
        ctx.save_for_backward(x, y, probs)
        return native_ops().silu_mul_probs_fwd(x, y, probs)

    @staticmethod
    def backward(ctx: Any, grad_output: torch.Tensor):  # type: ignore[override]
        x, y, probs = ctx.saved_tensors
        return native_ops().silu_mul_probs_bwd(contiguous_aligned(grad_output), x, y, probs)


def silu_mul_probs(x: torch.Tensor, y: torch.Tensor, probs: torch.Tensor) -> torch.Tensor:
    """``silu(x) * y * probs[:, None]`` for expert-sorted rows; ``probs`` is fp32 ``[rows]``."""
    if on_gpu(x):
        return SiLUMulProbsFunction.apply(x, y, probs.float())
    return (torch.nn.functional.silu(x.float()) * y.float() * probs.float()[:, None]).to(x.dtype)


__all__ = ["silu_mul", "silu_mul_probs", "silu_mul_reference"]
