"""CUDA path for attention: the hand-written wgmma flash-attention kernels (``ops/csrc/flash_attn.cu``).

Forward: one 128-row query tile per CTA (64 rows per consumer warpgroup) over K/V rings filled by TMA, S and O
accumulators in registers, P handed to the second GEMM as its register A operand, online softmax, LSE out.  Backward: delta pre-pass, a dK/dV
kernel (K,V resident, Q/dO streamed over the heads of the GQA group) and a dQ kernel (Q,dO resident, K/V streamed); no
atomics.  Causal / sliding window (left, right) / soft-cap / attention sinks / packed variable-length batches are all
handled inside the kernels.  There is no library (cuDNN / SDPA) call on this path.

Head dims (qk, v): (64, 64), (128, 128) and (192, 128), the last for multi-head latent attention (128 nope + 64 rope query /
key columns, 128 value columns); V, the output and dO keep their own width.

"""

from __future__ import annotations

import math

import torch

from .._native import native_ops


NATIVE_HEAD_DIMS = ((64, 64), (128, 128), (192, 128))  # (qk head dim, v head dim) pairs the kernels are built for


def native_supported(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor) -> bool:
    return (q.is_cuda and q.dtype == torch.bfloat16 and k.dtype == torch.bfloat16 and v.dtype == torch.bfloat16
            and (q.shape[-1], v.shape[-1]) in NATIVE_HEAD_DIMS and k.shape[-1] == q.shape[-1]
            and q.shape[-2] % k.shape[-2] == 0)


def _window(causal: bool, window_size: tuple[int | None, int | None]) -> tuple[int, int]:
    left, right = window_size
    wl = left if left is not None and left >= 0 else -1
    wr = 0 if causal else (right if right is not None and right >= 0 else -1)
    return wl, wr


class _NativeFlashAttention(torch.autograd.Function):
    """(q, k, v[, sink]) -> (out, lse); q/k are [B,S,H,Dqk], v / out [B,S,H,Dv], or packed [total,H,D] with ``cu_seqlens``."""

    @staticmethod
    def forward(ctx, q, k, v, sink, scale, wl, wr, softcap, cu_q, cu_k, max_q, max_k):
        ops = native_ops()
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        sink32 = sink.detach().float().contiguous() if sink is not None else None
        out, lse = ops.flash_attn_fwd(q, k, v, scale, wl, wr, softcap, sink32, cu_q, cu_k, max_q, max_k)
        ctx.save_for_backward(q, k, v, out, lse, sink, cu_q, cu_k)
        ctx.cfg = (scale, wl, wr, softcap, max_q, max_k)
        return out, lse

    @staticmethod
    def backward(ctx, dout, dlse):
        q, k, v, out, lse, sink, cu_q, cu_k = ctx.saved_tensors
        scale, wl, wr, softcap, max_q, max_k = ctx.cfg
        if dout is None:
            dout = torch.zeros_like(out)
        dlse32 = dlse.float().contiguous() if dlse is not None else None
        dq, dk, dv, delta = native_ops().flash_attn_bwd(dout.contiguous(), q, k, v, out, lse, scale, wl, wr, softcap, cu_q, cu_k,
                                                        max_q, max_k, dlse32)
        dsink = None
        if sink is not None and ctx.needs_input_grad[3]:
            # out_i = sum_j e^{a_ij} v_j / (L_i + e^s):  d/ds = -sum_{b,i} e^{s_h - lse} * (dout . out - dlse)
            # packed rows outside every sequence have lse = -inf and take no part
            sink_col = sink.float()[:, None] if lse.dim() == 2 else sink.float()[None, :, None]
            p_sink = torch.where(lse == -math.inf, 0.0, torch.exp(sink_col - lse))
            dsink = -(p_sink * delta).sum(dim=1 if lse.dim() == 2 else (0, 2)).to(sink.dtype)
        return dq, dk, dv, dsink, None, None, None, None, None, None, None, None


def flash_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, softmax_scale: float | None, causal: bool,
                    window_size: tuple[int | None, int | None] = (None, None), learnable_sink: torch.Tensor | None = None,
                    softcap: float = 0.0, cu_seqlens_q: torch.Tensor | None = None, cu_seqlens_k: torch.Tensor | None = None,
                    max_seqlen_q: int = 0, max_seqlen_k: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
    """``(out, lse)``; fixed-length: q ``[B,S,H,Dqk]``, out ``[B,S,H,Dv]``, lse ``[B,H,S]``; packed: q ``[total,H,Dqk]``,
    out ``[total,H,Dv]``, lse ``[H,total]``."""
    scale = float(softmax_scale) if softmax_scale is not None else 1.0 / math.sqrt(q.shape[-1])
    wl, wr = _window(causal, window_size)
    if cu_seqlens_q is not None:
        cu_seqlens_q = cu_seqlens_q.to(device=q.device, dtype=torch.int32).contiguous()
        cu_seqlens_k = cu_seqlens_k.to(device=q.device, dtype=torch.int32).contiguous()
    return _NativeFlashAttention.apply(q, k, v, learnable_sink, scale, wl, wr, float(softcap or 0.0), cu_seqlens_q, cu_seqlens_k,
                                       int(max_seqlen_q), int(max_seqlen_k))
