"""RMSNorm (reference kernels ``d9d/kernel/normalization/rms/op.py:6-266``; here: one register-resident pass,
128-bit vectorised, deterministic two-stage dw reduction instead of fp32 atomics)."""

from __future__ import annotations

from typing import Any

import torch
from torch.autograd import Function

from .._native import contiguous_aligned, native_ops, on_gpu


def rms_norm_reference(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, zero_centered: bool = False) -> torch.Tensor:
    """fp32 oracle."""
    xf = x.float()
    w = weight.float() + 1.0 if zero_centered else weight.float()
    out = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * w
    return out.to(x.dtype)


class RMSNormFunction(Function):
    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, weight: torch.Tensor, eps: float, zero_centered: bool) -> torch.Tensor:
        ops = native_ops()
        xc = contiguous_aligned(x)
        out, inv_rms = ops.rms_norm_fwd(xc, contiguous_aligned(weight), eps, zero_centered)
        ctx.save_for_backward(xc, weight, inv_rms)
        ctx.zero_centered = zero_centered
        return out

    @staticmethod
    def backward(ctx: Any, grad_output: torch.Tensor):  # type: ignore[override]
        x, weight, inv_rms = ctx.saved_tensors
        dx, dw = native_ops().rms_norm_bwd(contiguous_aligned(grad_output), x, contiguous_aligned(weight), inv_rms,
                                           ctx.zero_centered)
        return dx, dw, None, None


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, zero_centered: bool = False) -> torch.Tensor:
    """``x * rsqrt(mean(x^2) + eps) * (weight [+ 1])`` over the last dim, fp32 math, output in ``x.dtype``."""
    if on_gpu(x):
        if weight.dtype != x.dtype:
            weight = weight.to(x.dtype)
        return RMSNormFunction.apply(x, weight, eps, zero_centered)
    return rms_norm_reference(x, weight, eps, zero_centered)
