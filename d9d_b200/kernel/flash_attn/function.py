"""Attention entry points with the reference's ``flash_attn_func`` / ``flash_attn_varlen_func`` signatures
(``d9d/kernel/flash_attn/function.py:313-436``): causal, sliding window, GQA/MQA, softcap, learnable per-head
sinks (with analytic ``dsink``), optional LSE.

Backends:
* ``attention_reference``: exact fp32 math (CPU tensors; the oracle of the numerics tests),
* CUDA: the native wgmma flash-attention forward / backward kernels (``native.py``), every option in-kernel.
"""

from __future__ import annotations

import math

import torch


def _window_mask(sq: int, sk: int, causal: bool, window: tuple[int | None, int | None], device) -> torch.Tensor | None:
    left, right = window
    if not causal and left is None and right is None:
        return None
    # bottom-right aligned relative position (FlashAttention convention)
    qi = torch.arange(sq, device=device)[:, None] + (sk - sq)
    kj = torch.arange(sk, device=device)[None, :]
    keep = torch.ones(sq, sk, dtype=torch.bool, device=device)
    if causal:
        keep &= kj <= qi
    if left is not None and left >= 0:
        keep &= kj >= qi - left
    if right is not None and right >= 0 and not causal:
        keep &= kj <= qi + right
    return keep


def attention_reference(
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    softmax_scale: float | None = None,
    causal: bool = False,
    window_size: tuple[int | None, int | None] = (None, None),
    learnable_sink: torch.Tensor | None = None,
    softcap: float = 0.0,
) -> tuple[torch.Tensor, torch.Tensor]:
    """fp32 attention oracle. q: [B,Sq,H,D]; k/v: [B,Sk,Hk,D(v)]. Returns (out [B,Sq,H,Dv], lse [B,H,Sq])."""
    B, Sq, H, D = q.shape
    Sk, Hk = k.shape[1], k.shape[2]
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
    group = H // Hk
    qf = q.float().permute(0, 2, 1, 3)  # [B,H,Sq,D]
    kf = k.float().permute(0, 2, 1, 3).repeat_interleave(group, dim=1)
    vf = v.float().permute(0, 2, 1, 3).repeat_interleave(group, dim=1)
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    if softcap and softcap > 0:
        s = torch.tanh(s / softcap) * softcap
    keep = _window_mask(Sq, Sk, causal, window_size, q.device)
    if keep is not None:
        s = s.masked_fill(~keep, float("-inf"))
    if learnable_sink is not None:
        sink = learnable_sink.float().view(1, H, 1, 1).expand(B, H, Sq, 1)
        full = torch.cat([s, sink], dim=-1)
        lse = torch.logsumexp(full, dim=-1)
        p = torch.exp(s - lse.unsqueeze(-1))
    else:
        lse = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - lse.unsqueeze(-1))
    p = torch.nan_to_num(p, nan=0.0)
    out = torch.matmul(p, vf).permute(0, 2, 1, 3).to(q.dtype)
    return out, lse


_REFERENCE_SCORE_LIMIT = 1 << 22  # the fp32 oracle materialises [B,H,Sq,Sk]: test sizes only on a GPU


def _library_path_ok(q: torch.Tensor, k: torch.Tensor, causal, window_size, learnable_sink, softcap) -> bool:
    """Shapes / dtypes outside the native kernels (e.g. fp16, or qk / v head sizes the kernels are not built for): plain or
    causal attention goes to PyTorch SDPA (library flash kernels)."""
    if learnable_sink is not None or (softcap and softcap > 0):
        return False
    if window_size[0] is not None or window_size[1] is not None:
        return False
    return not (causal and q.shape[1] != k.shape[1])


def _sdpa(q, k, v, softmax_scale, causal):
    """SDPA's flash kernels need one head size: a narrower V is zero-padded to the qk head size and the output sliced back."""
    import torch.nn.functional as F

    dv = v.shape[-1]
    if dv < q.shape[-1]:
        v = F.pad(v, (0, q.shape[-1] - dv))
    qh, kh, vh = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    out = F.scaled_dot_product_attention(qh, kh, vh, is_causal=causal, scale=softmax_scale, enable_gqa=qh.shape[1] != kh.shape[1])
    out = out.transpose(1, 2)
    return out[..., :dv] if dv < q.shape[-1] else out


def flash_attn_func(
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    softmax_scale: float | None = None,
    causal: bool = False,
    window_size: tuple[int | None, int | None] = (None, None),
    learnable_sink: torch.Tensor | None = None,
    softcap: float = 0.0,
    num_splits: int = 1,
    pack_gqa: bool | None = None,
    deterministic: bool = False,
    return_lse: bool = False,
) -> tuple[torch.Tensor, torch.Tensor | None]:
    """Returns ``(output [B,S,H,Dv], lse [B,H,S] or None)``.

    CUDA bf16 tensors with (qk, v) head sizes (64, 64), (128, 128) or (192, 128) run the native wgmma kernels (forward
    and backward, every option); other CUDA inputs use SDPA for plain / causal attention (V zero-padded to the qk head
    size when it is narrower) and raise for options it cannot express - the fp32 oracle (which materialises the score
    matrix) is only taken on CPU or for tiny problems.
    """
    del num_splits, pack_gqa, deterministic  # the native backward is atomic-free: always deterministic
    if q.is_cuda:
        from .native import flash_attention, native_supported

        if native_supported(q, k, v):
            out, lse = flash_attention(q, k, v, softmax_scale, causal, window_size, learnable_sink, softcap)
            return out, (lse if return_lse else None)
        if not return_lse and _library_path_ok(q, k, causal, window_size, learnable_sink, softcap):
            return _sdpa(q, k, v, softmax_scale, causal), None
        if q.shape[0] * q.shape[2] * q.shape[1] * k.shape[1] > _REFERENCE_SCORE_LIMIT:
            raise NotImplementedError(
                f"attention with dtype {q.dtype}, head sizes {q.shape[-1]}/{v.shape[-1]} and these options has no fused CUDA "
                "path (native kernels: bf16, (qk, v) head sizes (64, 64), (128, 128) or (192, 128))")
    out, lse = attention_reference(q, k, v, softmax_scale, causal, window_size, learnable_sink, softcap)
    return out, (lse if return_lse else None)


def flash_attn_varlen_func(
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    cu_seqlens_q: torch.Tensor | None = None,
    cu_seqlens_k: torch.Tensor | None = None,
    max_seqlen_q: int | None = None,
    max_seqlen_k: int | None = None,
    seqused_q: torch.Tensor | None = None,
    seqused_k: torch.Tensor | None = None,
    page_table: torch.Tensor | None = None,
    softmax_scale: float | None = None,
    causal: bool = False,
    window_size: tuple[int | None, int | None] = (None, None),
    learnable_sink: torch.Tensor | None = None,
    softcap: float = 0.0,
    num_splits: int = 1,
    pack_gqa: bool | None = None,
    deterministic: bool = False,
    return_lse: bool = False,
) -> tuple[torch.Tensor, torch.Tensor | None]:
    """Packed variable-length attention: q ``[total_q, H, Dqk]``, k ``[total_k, Hk, Dqk]``, v ``[total_k, Hk, Dv]`` with
    ``cu_seqlens``; the output is ``[total_q, H, Dv]`` and the LSE ``[H, total_q]``.  On CUDA the sequence boundaries are resolved inside the kernels (no host synchronisation when
    ``max_seqlen_q`` / ``max_seqlen_k`` are given)."""
    del num_splits, pack_gqa, deterministic
    if page_table is not None or seqused_q is not None or seqused_k is not None:
        raise NotImplementedError("paged KV / seqused are not supported")
    if cu_seqlens_q is None or cu_seqlens_k is None:
        raise ValueError("cu_seqlens_q and cu_seqlens_k are required")
    if q.is_cuda:
        from .native import flash_attention, native_supported

        if native_supported(q, k, v):
            if max_seqlen_q is None:
                max_seqlen_q = int((cu_seqlens_q[1:] - cu_seqlens_q[:-1]).max())
            if max_seqlen_k is None:
                max_seqlen_k = int((cu_seqlens_k[1:] - cu_seqlens_k[:-1]).max())
            out, lse = flash_attention(q, k, v, softmax_scale, causal, window_size, learnable_sink, softcap, cu_seqlens_q,
                                       cu_seqlens_k, max_seqlen_q, max_seqlen_k)
            return out, (lse if return_lse else None)
    bq, bk = cu_seqlens_q.tolist(), cu_seqlens_k.tolist()
    outs, lses = [], []
    for i in range(len(bq) - 1):
        o, l = flash_attn_func(
            q[bq[i] : bq[i + 1]].unsqueeze(0), k[bk[i] : bk[i + 1]].unsqueeze(0), v[bk[i] : bk[i + 1]].unsqueeze(0),
            softmax_scale, causal, window_size, learnable_sink, softcap, return_lse=return_lse,
        )
        outs.append(o.squeeze(0))
        if return_lse:
            lses.append(l.squeeze(0))
    out = torch.cat(outs, dim=0)
    return out, (torch.cat(lses, dim=-1) if return_lse else None)
