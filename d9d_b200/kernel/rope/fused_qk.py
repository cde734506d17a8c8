"""Per-head q/k RMSNorm fused with rotary embedding (one launch forward, two backward; ``ops/csrc/qk_norm_rope.cu``)."""

from __future__ import annotations

from typing import Any

import torch
from torch.autograd import Function

from .._native import contiguous_aligned, native_ops, on_gpu


def _heads_aligned(x: torch.Tensor) -> torch.Tensor:
    """[T, H, D] with dense heads, its base and token stride 16-byte aligned (the kernel moves 8 bf16 per access); a view
    that is not is copied into a fresh buffer."""
    if x.stride(2) == 1 and x.stride(1) == x.shape[2] and x.data_ptr() % 16 == 0 and x.stride(0) % 8 == 0:
        return x
    return x.clone(memory_format=torch.contiguous_format)


class _QkNormRope(Function):
    @staticmethod
    def forward(ctx: Any, q: torch.Tensor, k: torch.Tensor, wq: torch.Tensor, wk: torch.Tensor, cos_t: torch.Tensor,
                sin_t: torch.Tensor, eps: float, zero_centered: bool, style: int):
        q3 = _heads_aligned(q.reshape(-1, q.shape[-2], q.shape[-1]))
        k3 = _heads_aligned(k.reshape(-1, k.shape[-2], k.shape[-1]))
        wq, wk = contiguous_aligned(wq), contiguous_aligned(wk)
        qo, ko, inv = native_ops().qk_norm_rope_fwd(q3, k3, wq, wk, cos_t, sin_t, eps, zero_centered, style)
        ctx.save_for_backward(q3, k3, wq, wk, cos_t, sin_t, inv)
        ctx.zero_centered, ctx.style, ctx.q_shape, ctx.k_shape = zero_centered, style, q.shape, k.shape
        return qo.view(q.shape), ko.view(k.shape)

    @staticmethod
    def backward(ctx: Any, dqo: torch.Tensor, dko: torch.Tensor):  # type: ignore[override]
        q3, k3, wq, wk, cos_t, sin_t, inv = ctx.saved_tensors
        dqo, dko = contiguous_aligned(dqo.reshape(q3.shape)), contiguous_aligned(dko.reshape(k3.shape))
        dq, dk, dwq, dwk = native_ops().qk_norm_rope_bwd(dqo, dko, q3, k3, wq, wk, cos_t, sin_t, inv, ctx.zero_centered,
                                                         ctx.style)
        return dq.view(ctx.q_shape), dk.view(ctx.k_shape), dwq.to(wq.dtype), dwk.to(wk.dtype), None, None, None, None, None


def fused_qk_norm_rope_supported(q: torch.Tensor, k: torch.Tensor, wq: torch.Tensor, wk: torch.Tensor, rope_dim: int) -> bool:
    d = q.shape[-1]
    return (on_gpu(q) and q.dtype == torch.bfloat16 and k.dtype == torch.bfloat16 and wq.dtype == torch.bfloat16
            and wk.dtype == torch.bfloat16 and d in (64, 128, 256) and k.shape[-1] == d and rope_dim <= d
            and rope_dim % 16 == 0)


def qk_norm_rope(q: torch.Tensor, k: torch.Tensor, wq: torch.Tensor, wk: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor,
                 eps: float, zero_centered: bool, style: int) -> tuple[torch.Tensor, torch.Tensor]:
    """``q [..., Hq, D]``, ``k [..., Hk, D]`` (views of the projection outputs are fine), ``cos/sin [..., rope_dim]``
    per token -> normalised and rotated ``q, k`` (contiguous)."""
    rope_dim = cos.shape[-1]
    cos_t = contiguous_aligned(cos.reshape(-1, rope_dim).float())
    sin_t = contiguous_aligned(sin.reshape(-1, rope_dim).float())
    return _QkNormRope.apply(q, k, wq, wk, cos_t, sin_t, eps, zero_centered, style)
