from __future__ import annotations

import torch
from torch import nn

from d9d_b200.module.base import ModuleLateInit
from d9d_b200.module.block.attention.sdpa import FlashSdpa
from d9d_b200.module.block.linear import Linear
from d9d_b200.module.block.normalization import RMSNorm
from d9d_b200.module.block.positional import RotaryEmbeddingApplicator, RotaryEmbeddingStyle


class LowRankProjection(nn.Module, ModuleLateInit):
    """``up(norm(down(x)))`` bottleneck projection."""

    def __init__(self, in_features: int, bottleneck: int, out_features: int, norm_eps: float):
        super().__init__()
        self.down_proj = Linear(in_features, bottleneck, bias=False)
        self.norm = RMSNorm(bottleneck, eps=norm_eps)
        self.up_proj = Linear(bottleneck, out_features, bias=False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.up_proj(self.norm(self.down_proj(x)))

    def reset_parameters(self) -> None:
        self.down_proj.reset_parameters()
        self.norm.reset_parameters()
        self.up_proj.reset_parameters()


class MultiHeadLatentAttention(nn.Module, ModuleLateInit):
    """DeepSeek-V2 multi-head latent attention (reference ``d9d/module/block/attention/multi_head_latent.py:11-220``):
    low-rank KV latent + shared rotary key, decoupled nope/rope query parts.  V keeps its own head dim: the attention
    kernels take qk and v head dims separately (the native CUDA kernels at (192, 128), DeepSeek-V2 / V3's dims).
    """

    def __init__(self, hidden_size: int, num_attention_heads: int, qk_nope_head_dim: int, qk_rope_head_dim: int,
                 v_head_dim: int, kv_lora_rank: int, q_lora_rank: int | None, qk_down_norm_eps: float,
                 is_causal: bool, rope_style: RotaryEmbeddingStyle):
        super().__init__()
        self._n_heads = num_attention_heads
        self._nope = qk_nope_head_dim
        self._rope = qk_rope_head_dim
        self._qk = qk_nope_head_dim + qk_rope_head_dim
        self._v = v_head_dim
        self._kv_rank = kv_lora_rank
        self._q_lora_rank = q_lora_rank
        self._scaling = self._qk**-0.5
        self._is_causal = is_causal
        if v_head_dim > self._qk:
            raise ValueError(f"v_head_dim ({v_head_dim}) must not exceed qk_head_dim ({self._qk}).")

        if q_lora_rank is not None:
            self.q_proj: nn.Module = LowRankProjection(hidden_size, q_lora_rank, num_attention_heads * self._qk, qk_down_norm_eps)
        else:
            self.q_proj = Linear(hidden_size, num_attention_heads * self._qk, bias=False)
        self.kv_down_proj = Linear(hidden_size, kv_lora_rank + qk_rope_head_dim, bias=False)
        self.kv_down_norm = RMSNorm(kv_lora_rank, eps=qk_down_norm_eps)
        self.kv_up_proj = Linear(kv_lora_rank, num_attention_heads * (qk_nope_head_dim + v_head_dim), bias=False)
        self.o_proj = Linear(num_attention_heads * v_head_dim, hidden_size, bias=False)
        self.rope = RotaryEmbeddingApplicator(style=rope_style)
        self.kernel = FlashSdpa()

    @property
    def q_lora_rank(self) -> int | None:
        return self._q_lora_rank

    def forward(self, hidden_states: torch.Tensor, attention_mask: torch.Tensor | None,
                position_embeddings: tuple[torch.Tensor, torch.Tensor]) -> torch.Tensor:
        b, s, _ = hidden_states.shape
        cos, sin = position_embeddings
        h = self._n_heads

        q = self.q_proj(hidden_states).view(b, s, h, self._qk)
        q_nope, q_rope = q.split([self._nope, self._rope], dim=-1)

        kv = self.kv_down_proj(hidden_states)
        latent, k_rope = kv.split([self._kv_rank, self._rope], dim=-1)
        kv_up = self.kv_up_proj(self.kv_down_norm(latent.contiguous())).view(b, s, h, self._nope + self._v)
        k_nope, v = kv_up.split([self._nope, self._v], dim=-1)

        k_rope = k_rope.unsqueeze(2)  # one rotary key shared by every head
        q_rope, k_rope = self.rope(q_rope.contiguous(), k_rope.contiguous(), cos, sin)
        q = torch.cat([q_nope, q_rope], dim=-1)
        k = torch.cat([k_nope, k_rope.expand(-1, -1, h, -1)], dim=-1)

        out = self.kernel(q, k, v, attention_mask=attention_mask, is_causal=self._is_causal, scale=self._scaling)
        return self.o_proj(out.reshape(b, s, h * self._v))

    def reset_parameters(self) -> None:
        for mod in (self.q_proj, self.kv_down_proj, self.kv_down_norm, self.kv_up_proj, self.o_proj):
            mod.reset_parameters()
