"""Dense linear layers on the hand-written wgmma GEMM (TMA-fed, register accumulators, persistent, warp-specialised).

* forward   ``y = x @ W^T``                       K-major A and B
* dgrad     ``dx = dy @ W``                       B consumed MN-major straight from ``W[out, in]`` (no transpose)
* wgrad     ``dW = dy^T @ x``                     both operands consumed MN-major; fp32 or bf16 output, optional
                                                   accumulation into an existing gradient buffer in the epilogue
Split backward (zero-bubble PP) is honoured through ``GLOBAL_GRAD_CONTEXT``.
"""

from __future__ import annotations

from typing import Any

import torch
from torch.autograd import Function

from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection

from .._native import fused_wgrad_buffer, fused_wgrad_owner, grad_dtype_of, native_ops, on_gpu


def _tma_ok(*tensors: torch.Tensor) -> bool:
    for t in tensors:
        if t.dtype != torch.bfloat16 or t.dim() != 2 or t.stride(1) != 1:
            return False
        if t.data_ptr() % 16 or (t.stride(0) * 2) % 16:
            return False
    return True


def gemm_nt(a: torch.Tensor, b: torch.Tensor, out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``a[M,K] @ b[N,K]^T`` on the native GEMM."""
    out = torch.empty(a.shape[0], b.shape[0], device=a.device, dtype=out_dtype)
    native_ops().gemm(a, b, out, False, False, False)
    return out


class LinearFunction(Function):
    """``y = x @ W^T``.  ``owner`` (optional) is the leaf parameter whose pre-allocated gradient buffer receives
    ``dW`` directly from the wgrad GEMM epilogue (see ``fused_wgrad_owner``); ``weight`` is then passed detached."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, weight: torch.Tensor, owner: torch.Tensor | None = None) -> torch.Tensor:
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        ctx.save_for_backward(x2, weight)
        ctx.x_shape = x.shape
        ctx.owner = owner
        out = torch.empty(x2.shape[0], weight.shape[0], device=x.device, dtype=x.dtype)
        native_ops().gemm(x2, weight, out, False, False, False)
        return out.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx: Any, grad_output: torch.Tensor):  # type: ignore[override]
        x2, weight = ctx.saved_tensors
        dy = grad_output.reshape(-1, grad_output.shape[-1])
        if not dy.is_contiguous():
            dy = dy.contiguous()
        ops = native_ops()
        dx = dw = None
        if ctx.needs_input_grad[0] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.inputs):
            dx = torch.empty_like(x2)
            ops.gemm(dy, weight, dx, False, True, False)  # dy[M,out] @ W[out,in]
            dx = dx.view(ctx.x_shape)
        if GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.weight):
            if ctx.owner is not None and ctx.needs_input_grad[2]:
                ops.gemm(dy, x2, fused_wgrad_buffer(ctx.owner), True, True, True)  # grad += dy^T @ x in the epilogue
            elif ctx.needs_input_grad[1]:
                dw = torch.empty(weight.shape, device=weight.device, dtype=grad_dtype_of(weight))
                ops.gemm(dy, x2, dw, True, True, False)  # dy^T[out,M] @ x[M,in]
        return dx, dw, None


def linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None = None) -> torch.Tensor:
    """``x @ weight^T (+ bias)``; native wgmma path for bf16 CUDA tensors, ``F.linear`` on CPU."""
    if on_gpu(x) and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16:
        x2 = x.reshape(-1, x.shape[-1])
        if _tma_ok(weight) and x2.shape[-1] % 8 == 0 and weight.shape[0] % 8 == 0 and x2.numel() > 0:
            owner = fused_wgrad_owner(weight)
            out = LinearFunction.apply(x, weight, None) if owner is None else LinearFunction.apply(x, weight.detach(), owner)
            return out if bias is None else out + bias
        raise RuntimeError(
            f"d9d_b200.linear: operand layout not supported by the native GEMM (x {tuple(x.shape)}, W {tuple(weight.shape)})"
        )
    return torch.nn.functional.linear(x, weight, bias)


__all__ = ["LinearFunction", "gemm_nt", "linear"]
