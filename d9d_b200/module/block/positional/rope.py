"""Rotary embeddings (reference ``d9d/module/block/positional/rope.py:10-216``).

Difference from the reference: the applicator is one fused kernel per tensor (``d9d_b200.kernel.rope``) instead of eager
``q*cos + rotate(q)*sin``; cos/sin caches are kept in fp32.
"""

from __future__ import annotations

import enum

import torch
from torch import nn

from d9d_b200.kernel import rope as rope_kernel
from d9d_b200.kernel._native import native_ops, on_gpu
from d9d_b200.module.base import ModuleLateInit

from .rope_scaling import NoRopeScaling, RopeScaling


class RotaryEmbeddingStyle(enum.StrEnum):
    HALF = "half"  # pairs are (i, i + d/2)
    INTERLEAVED = "interleaved"  # pairs are (2i, 2i + 1)


def _style_code(style: RotaryEmbeddingStyle) -> int:
    if style == RotaryEmbeddingStyle.HALF:
        return rope_kernel.STYLE_HALF
    if style == RotaryEmbeddingStyle.INTERLEAVED:
        return rope_kernel.STYLE_INTERLEAVED
    raise ValueError(f"Unknown RoPE style: {style}")


def prepare_rotary_cos_sin_emb(
    rope_base: int,
    head_dim: int,
    max_position_ids: int,
    device: torch.device,
    dtype: torch.dtype,
    style: RotaryEmbeddingStyle,
    rope_scaling: RopeScaling | None = None,
) -> tuple[torch.Tensor, torch.Tensor]:
    """``cos/sin [max_position_ids, head_dim]`` laid out for ``style`` and multiplied by the scaling's mscale."""
    scaling = rope_scaling if rope_scaling is not None else NoRopeScaling()
    inv_freq = scaling.inverse_frequencies(rope_base, head_dim).float()
    angles = torch.outer(torch.arange(max_position_ids, dtype=torch.float32), inv_freq)
    if style == RotaryEmbeddingStyle.HALF:
        table = torch.cat((angles, angles), dim=-1)
    elif style == RotaryEmbeddingStyle.INTERLEAVED:
        table = angles.repeat_interleave(2, dim=-1)
    else:
        raise ValueError(f"Unknown RoPE style: {style}")
    mscale = scaling.attention_mscale
    return (table.cos() * mscale).to(device=device, dtype=dtype), (table.sin() * mscale).to(device=device, dtype=dtype)


class RotaryEmbeddingProvider(nn.Module, ModuleLateInit):
    """Caches cos/sin for every position up to ``max_position_ids`` and serves them by ``position_ids``."""

    def __init__(self, rope_base: int, head_dim: int, max_position_ids: int, style: RotaryEmbeddingStyle,
                 rope_scaling: RopeScaling | None = None) -> None:
        super().__init__()
        self._rope_base = rope_base
        self._head_dim = head_dim
        self._max_position_ids = max_position_ids
        self._style = style
        self._rope_scaling = rope_scaling if rope_scaling is not None else NoRopeScaling()
        self.cos_emb = nn.Buffer(torch.empty(max_position_ids, head_dim), persistent=False)
        self.sin_emb = nn.Buffer(torch.empty(max_position_ids, head_dim), persistent=False)

    def forward(self, position_ids: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        return self.cos_emb[position_ids], self.sin_emb[position_ids]

    def reset_parameters(self) -> None:
        with torch.no_grad():
            # the angle tables stay fp32 even when the model is cast to bf16: they feed fp32 math in the kernel
            cos, sin = prepare_rotary_cos_sin_emb(
                self._rope_base, self._head_dim, self._max_position_ids, self.cos_emb.device, torch.float32,
                self._style, self._rope_scaling,
            )
            self.cos_emb.data = cos
            self.sin_emb.data = sin


class RotaryEmbeddingApplicator(nn.Module):
    """Rotates q and k (layout ``[B, S, heads, dim]``) by cos/sin of shape ``[B, S, dim]``."""

    def __init__(self, style: RotaryEmbeddingStyle) -> None:
        super().__init__()
        self._style = style
        self._code = _style_code(style)

    @property
    def style_code(self) -> int:
        return self._code

    def _rotate(self, x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
        if on_gpu(x) and x.dtype == torch.bfloat16 and x.shape[-1] % 64 == 0:
            rope_dim = cos.shape[-1]
            cos2 = cos.reshape(-1, rope_dim).float().contiguous()
            sin2 = sin.reshape(-1, rope_dim).float().contiguous()
            return _IdentityPosRope.apply(x, cos2, sin2, self._code)
        return rope_kernel.rotate_reference(x, cos, sin, self._code)

    def forward(self, query_states: torch.Tensor, key_states: torch.Tensor, position_embedding_cos: torch.Tensor,
                position_embedding_sin: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        return (self._rotate(query_states, position_embedding_cos, position_embedding_sin),
                self._rotate(key_states, position_embedding_cos, position_embedding_sin))


class _IdentityPosRope(torch.autograd.Function):
    """RoPE kernel fed with already-gathered per-token cos/sin (position index == token index)."""

    @staticmethod
    def forward(ctx, x, cos2, sin2, style):
        shape = x.shape
        x3 = x.reshape(-1, shape[-2], shape[-1])
        if x3.stride(2) != 1 or x3.stride(1) != shape[-1]:
            x3 = x3.contiguous()
        pos = torch.arange(x3.shape[0], device=x.device, dtype=torch.long)
        ctx.save_for_backward(cos2, sin2, pos)
        ctx.style = style
        return native_ops().rope_apply(x3, cos2, sin2, pos, style, False).view(shape)

    @staticmethod
    def backward(ctx, grad_output):
        cos2, sin2, pos = ctx.saved_tensors
        shape = grad_output.shape
        g3 = grad_output.reshape(-1, shape[-2], shape[-1]).contiguous()
        return native_ops().rope_apply(g3, cos2, sin2, pos, ctx.style, True).view(shape), None, None, None
