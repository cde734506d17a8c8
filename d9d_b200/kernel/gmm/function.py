"""Grouped GEMM with the reference's ``gmm`` signature (``d9d/kernel/gmm/function.py:10-76``).

The reference delegates to the ``grouped_gemm`` wheel and needs ``batch_sizes`` on the CPU.  This compatibility
entry keeps that contract (arbitrary group sizes) by re-packing rows into the 128-row aligned layout the native
wgmma grouped GEMM works on; the model path (``GroupedSwiGLU``) uses the aligned layout end-to-end and never
comes through here.
"""

from __future__ import annotations

from typing import Any

import torch
from torch.autograd import Function

from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection

from .._native import native_ops, on_gpu

_ALIGN = 128


def _aligned_plan(batch_sizes: torch.Tensor, device: torch.device):
    sizes = [int(s) for s in batch_sizes.tolist()]
    src_rows, dst_rows, seg, tiles = [], [], [0], []
    src = 0
    for e, n in enumerate(sizes):
        start = seg[-1]
        padded = (n + _ALIGN - 1) // _ALIGN * _ALIGN
        src_rows.extend(range(src, src + n))
        dst_rows.extend(range(start, start + n))
        tiles.extend([e] * (padded // _ALIGN))
        seg.append(start + padded)
        src += n
    cap = max(seg[-1], _ALIGN)
    tiles.extend([-1] * (cap // _ALIGN - len(tiles)))
    return (
        torch.tensor(src_rows, dtype=torch.long, device=device),
        torch.tensor(dst_rows, dtype=torch.long, device=device),
        torch.tensor(seg, dtype=torch.int32, device=device),
        torch.tensor(tiles, dtype=torch.int32, device=device),
        cap,
    )


def _gmm_reference(a, b, batch_sizes, trans_a=False, trans_b=False):
    sizes = [int(s) for s in batch_sizes.tolist()]
    outs, start = [], 0
    for e, n in enumerate(sizes):
        rows = a[start : start + n]
        if trans_a:
            outs.append(rows.t() @ b[start : start + n])
        else:
            outs.append(rows @ (b[e].t() if trans_b else b[e]))
        start += n
    return torch.stack(outs) if trans_a else torch.cat(outs, dim=0)


def _pad_rows(x: torch.Tensor, src: torch.Tensor, dst: torch.Tensor, cap: int) -> torch.Tensor:
    out = x.new_zeros(cap, x.shape[1])
    out.index_copy_(0, dst, x.index_select(0, src))
    return out


class GroupedGemm(Function):
    @staticmethod
    def forward(ctx: Any, a, b, batch_sizes, a_grad_direction, b_grad_direction, trans_b):
        ctx.save_for_backward(a, b, batch_sizes)
        ctx.dirs = (a_grad_direction, b_grad_direction)
        ctx.trans_b = trans_b
        if not on_gpu(a):
            return _gmm_reference(a, b, batch_sizes, trans_b=trans_b)
        src, dst, seg, tiles, cap = _aligned_plan(batch_sizes, a.device)
        ctx.plan = (src, dst, seg, tiles, cap)
        ap = _pad_rows(a, src, dst, cap)
        n_out = b.shape[1] if trans_b else b.shape[2]
        outp = torch.empty(cap, n_out, device=a.device, dtype=a.dtype)
        native_ops().gemm_grouped_m(ap, b.contiguous(), outp, tiles, not trans_b)
        out = a.new_empty(a.shape[0], n_out)
        out.index_copy_(0, src, outp.index_select(0, dst))
        return out

    @staticmethod
    def backward(ctx: Any, grad: torch.Tensor):  # type: ignore[override]
        a, b, batch_sizes = ctx.saved_tensors
        a_dir, b_dir = ctx.dirs
        trans_b = ctx.trans_b
        need_a = ctx.needs_input_grad[0] and GLOBAL_GRAD_CONTEXT.check_direction(a_dir)
        need_b = ctx.needs_input_grad[1] and GLOBAL_GRAD_CONTEXT.check_direction(b_dir)
        da = db = None
        if not on_gpu(a):
            if need_a:
                da = _gmm_reference(grad, b, batch_sizes, trans_b=not trans_b)
            if need_b:
                db = _gmm_reference(grad, a, batch_sizes, trans_a=True) if trans_b else _gmm_reference(a, grad, batch_sizes, trans_a=True)
            return da, db, None, None, None, None
        src, dst, seg, tiles, cap = ctx.plan
        ops = native_ops()
        gp = _pad_rows(grad.contiguous(), src, dst, cap)
        if need_a:
            dap = torch.empty(cap, a.shape[1], device=a.device, dtype=a.dtype)
            ops.gemm_grouped_m(gp, b.contiguous(), dap, tiles, trans_b)
            da = a.new_empty(a.shape)
            da.index_copy_(0, src, dap.index_select(0, dst))
        if need_b:
            ap = _pad_rows(a, src, dst, cap)
            db = torch.empty(b.shape, device=b.device, dtype=b.dtype)
            if trans_b:  # b: [E, N, K]  -> db[e] = grad_e^T @ a_e
                ops.gemm_grouped_k(gp, ap, db, seg, False)
            else:  # b: [E, K, N]  -> db[e] = a_e^T @ grad_e
                ops.gemm_grouped_k(ap, gp, db, seg, False)
        return da, db, None, None, None, None


def gmm(
    a: torch.Tensor,
    b: torch.Tensor,
    batch_sizes: torch.Tensor,
    a_grad_direction: GradDirection | None,
    b_grad_direction: GradDirection | None,
    trans_b: bool = False,
) -> torch.Tensor:
    """``out[rows of group e] = a[rows of group e] @ (b[e]^T if trans_b else b[e])``; ``batch_sizes`` lives on the CPU."""
    return GroupedGemm.apply(a, b, batch_sizes, a_grad_direction, b_grad_direction, trans_b)
