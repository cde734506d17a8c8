"""The whole expert block ``probs * down(silu(gate(x)) * up(x))`` over the 128-row aligned layout as ONE autograd node.

Compared with composing ``grouped_linear`` / ``silu_mul_probs`` nodes this
* lets the two input-gradient GEMMs (gate, up) accumulate into one buffer in their epilogues (no separate add pass),
* limits the element-wise kernels to the rows that are really in use (static-capacity buffers of the expert-parallel path
  are mostly empty),
* lets the caller name the buffers the block writes its output / input gradient into - the expert-parallel handler passes
  its NVLink-mapped staging region, so the peers read the results in place (no staging copies),
* honours split backward passes (``GLOBAL_GRAD_CONTEXT``): the input pass stashes what the weight pass needs.

The node takes its GEMMs as an argument: :class:`_Bf16ExpertGemms` (bf16 wgmma grouped GEMMs),
:class:`_Fp8ExpertGemms` (e4m3 grouped GEMMs with per-expert row / column scales, operands quantised per call) or
:class:`_BlockwiseFp8ExpertGemms` (DeepSeek-V3's blockwise recipe: 1x128 / 128x128 scales, promoted per k-block).

Reference: ``d9d/module/block/moe/grouped_experts.py:36-73`` (three ``gmm`` calls + ``silu_mul`` + a probability multiply).
"""

from __future__ import annotations

import functools
from typing import Any

import torch
from torch.autograd import Function

from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection

from .._native import fused_wgrad_buffer, fused_wgrad_owner, grad_dtype_of, native_ops
from ..fp8 import (
    blockwise_mm_reference,
    quantize_blockwise_reference,
    quantize_blockwise_t_reference,
    quantize_colwise_t_reference,
    quantize_rowwise_reference,
    quantize_weight_blocks_reference,
)
from .layout import MoELayout


class _Bf16ExpertGemms:
    """The block's GEMMs on bf16 operands.  ``rows`` / ``cols`` prepare an activation once for the GEMMs that read it
    row-wise (forward, input gradient) / along the tokens (weight gradient)."""

    @staticmethod
    def rows(ops, x, layout: MoELayout):
        return x

    cols = rows

    @staticmethod
    def fwd(ops, a, w, out, layout: MoELayout):  # out = a @ W[e]
        ops.gemm_grouped_m(a, w, out, layout.tile_group, True)

    @staticmethod
    def dgrad(ops, a, w, out, layout: MoELayout, accumulate: bool):  # out (+)= a @ W[e]^T, W[e] read as [N' = in, K' = out]
        ops.gemm_grouped_m(a, w, out, layout.tile_group, False, accumulate)

    @staticmethod
    def wgrad(ops, x, dy, out, layout: MoELayout, accumulate: bool):  # out[e] (+)= x_e^T dy_e
        ops.gemm_grouped_k(x, dy, out, layout.seg_offsets, accumulate)


class _Fp8ExpertGemms:
    """The block's GEMMs in e4m3 with fp32 row / column scales (the weights stay bf16 and are quantised per call):

    forward  ``y  = Q_row(x)  · Q_colT(W[e])``   scales: token x (expert, out)
    dgrad    ``dx = Q_row(dy) · Q_row(W[e])^T``  scales: token x (expert, in)
    wgrad    ``dW[e] = Q_seg(x)_e^T · Q_seg(dy)_e`` both transposed per expert segment, scales (expert, in) x (expert, out)
    """

    @staticmethod
    def rows(ops, x, layout: MoELayout):
        return ops.quantize_rowwise(x)

    @staticmethod
    def cols(ops, x, layout: MoELayout):
        return ops.quantize_segments_t(x, layout.tile_group, layout.seg_offsets, layout.counts)

    @staticmethod
    def fwd(ops, a, w, out, layout: MoELayout):
        wq, sw = ops.quantize_colwise_t_batched(w)  # [E, out, in], scale per (expert, out)
        ops.gemm_fp8_grouped_m(a[0], a[1], wq, sw, out, layout.tile_group, False)

    @staticmethod
    def dgrad(ops, a, w, out, layout: MoELayout, accumulate: bool):
        E, n_in, n_out = w.shape
        wq, sw = ops.quantize_rowwise(w.reshape(E * n_in, n_out))  # [E, in, out], scale per (expert, in)
        ops.gemm_fp8_grouped_m(a[0], a[1], wq.view(E, n_in, n_out), sw, out, layout.tile_group, accumulate)

    @staticmethod
    def wgrad(ops, x, dy, out, layout: MoELayout, accumulate: bool):
        ops.gemm_fp8_grouped_k(x[0], x[1], dy[0], dy[1], out, layout.seg_offsets, accumulate)


class _BlockwiseFp8ExpertGemms:
    """The block's GEMMs in e4m3 under DeepSeek-V3's blockwise recipe (weights stay bf16, quantised per call); every
    128-deep k-block is promoted into the fp32 accumulator with its own scales:

    forward  ``y  = Q_1x128(x)  · Q_128x128(W[e])``     activation scale per (token, 128 inputs), weight per 128x128 block
    dgrad    ``dx = Q_1x128(dy) · Q_128x128(W[e])^T``   the same weight blocks, in the copy that reduces over ``out``
    wgrad    ``dW[e] = Q_128t(x)_e^T · Q_128t(dy)_e``   per (128-token group, channel); the groups start at every
             expert's first row, so none straddles two experts and an outlier token sets the scale of its own group only
    """

    @staticmethod
    def rows(ops, x, layout: MoELayout):
        return ops.quantize_blockwise_tiles(x, layout.tile_group)

    @staticmethod
    def cols(ops, x, layout: MoELayout):
        return ops.quantize_blockwise_t_tiles(x, layout.tile_group, layout.seg_offsets, layout.counts)

    @staticmethod
    def fwd(ops, a, w, out, layout: MoELayout):
        wq, sw = ops.quantize_expert_weight_blocks(w, True)  # [E, out, in], scales [E, ceil(in/128), out]
        ops.gemm_fp8_blockwise_grouped_m(a[0], a[1], wq, sw, out, layout.tile_group, False)

    @staticmethod
    def dgrad(ops, a, w, out, layout: MoELayout, accumulate: bool):
        wq, sw = ops.quantize_expert_weight_blocks(w, False)  # [E, in, out], scales [E, ceil(out/128), in]
        ops.gemm_fp8_blockwise_grouped_m(a[0], a[1], wq, sw, out, layout.tile_group, accumulate)

    @staticmethod
    def wgrad(ops, x, dy, out, layout: MoELayout, accumulate: bool):
        ops.gemm_fp8_blockwise_grouped_k(x[0], x[1], dy[0], dy[1], out, layout.seg_offsets, accumulate)


_FP8_EXPERT_GEMMS = {"rowwise": _Fp8ExpertGemms, "blockwise": _BlockwiseFp8ExpertGemms}
FP8_EXPERT_RECIPES = tuple(_FP8_EXPERT_GEMMS)


def _check_fp8_recipe(recipe: str) -> None:
    if recipe not in _FP8_EXPERT_GEMMS:
        raise ValueError(f"unknown fp8 expert recipe {recipe!r} (expected one of {FP8_EXPERT_RECIPES})")


def _wgrad(ops, gemms, x_cols, dy: torch.Tensor, weight: torch.Tensor, owner: torch.Tensor | None, layout: MoELayout,
           needs_weight: bool, needs_owner: bool) -> torch.Tensor | None:
    """dW[e] (+)= x_e^T dy_e; accumulates straight into the owner's pre-allocated gradient when there is one.  The operands
    are prepared (``x_cols()``, ``gemms.cols(dy)``: the fp8 transposing quantisers) only when a gradient is wanted."""
    fused = owner is not None and needs_owner
    if not fused and not needs_weight:
        return None
    x, dy = x_cols(), gemms.cols(ops, dy, layout)
    if fused:
        gemms.wgrad(ops, x, dy, fused_wgrad_buffer(owner), layout, True)
        return None
    dw = torch.empty(weight.shape, device=weight.device, dtype=grad_dtype_of(weight))
    gemms.wgrad(ops, x, dy, dw, layout, False)
    return dw


class _GroupedSwiGLUFunction(Function):
    @staticmethod
    def forward(ctx: Any, xp, pp, wg, wu, wd, layout: MoELayout, og, ou, od, out_buf, dx_buf, gemms=_Bf16ExpertGemms):
        ops = native_ops()
        cap, ffn = xp.shape[0], wg.shape[2]
        valid = layout.seg_offsets[-1:]  # device scalar: rows in use
        gate = torch.empty(cap, ffn, device=xp.device, dtype=xp.dtype)
        up = torch.empty(cap, ffn, device=xp.device, dtype=xp.dtype)
        a = gemms.rows(ops, xp, layout)
        gemms.fwd(ops, a, wg, gate, layout)
        gemms.fwd(ops, a, wu, up, layout)
        h = ops.silu_mul_probs_fwd(gate, up, pp, valid)
        y = out_buf[:cap] if out_buf is not None else torch.empty(cap, wd.shape[2], device=xp.device, dtype=xp.dtype)
        gemms.fwd(ops, gemms.rows(ops, h, layout), wd, y, layout)
        ctx.save_for_backward(xp, pp, gate, up, h, wg, wu, wd)
        ctx.layout, ctx.owners, ctx.dx_buf, ctx.stash, ctx.gemms = layout, (og, ou, od), dx_buf, None, gemms
        return y

    @staticmethod
    def backward(ctx: Any, dy: torch.Tensor):  # type: ignore[override]
        xp, pp, gate, up, h, wg, wu, wd = ctx.saved_tensors
        layout: MoELayout = ctx.layout
        og, ou, od = ctx.owners
        gemms = ctx.gemms
        ops = native_ops()
        do_inputs = GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.inputs)
        do_weights = GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.weight)
        valid = layout.seg_offsets[-1:]
        cap = xp.shape[0]

        if ctx.stash is not None:  # weight pass of a split backward: the input pass left what we need
            dy, dgate, dup = ctx.stash
            ctx.stash = None
        else:
            dy = dy.contiguous()
            dh = torch.empty(cap, wd.shape[1], device=xp.device, dtype=xp.dtype)
            gemms.dgrad(ops, gemms.rows(ops, dy, layout), wd, dh, layout, False)
            dgate = dup = None

        dwd = dwg = dwu = dxp = dpp = None
        if do_weights:
            dwd = _wgrad(ops, gemms, lambda: gemms.cols(ops, h, layout), dy, wd, od, layout, ctx.needs_input_grad[4],
                         ctx.needs_input_grad[8])
        if dgate is None:
            dgate, dup, dpp = ops.silu_mul_probs_bwd(dh, gate, up, pp, valid)
        if do_inputs and (ctx.needs_input_grad[0] or ctx.needs_input_grad[1]):
            if ctx.needs_input_grad[0]:
                whole = do_weights  # a split backward reads dy again later: never alias the caller's staging buffers then
                dxp = ctx.dx_buf[:cap] if (ctx.dx_buf is not None and whole) else torch.empty_like(xp)
                gemms.dgrad(ops, gemms.rows(ops, dgate, layout), wg, dxp, layout, False)
                gemms.dgrad(ops, gemms.rows(ops, dup, layout), wu, dxp, layout, True)  # += in the epilogue
        if do_weights:
            xc = functools.cache(lambda: gemms.cols(ops, xp, layout))  # shared by the gate and up gradients
            dwg = _wgrad(ops, gemms, xc, dgate, wg, og, layout, ctx.needs_input_grad[2], ctx.needs_input_grad[6])
            dwu = _wgrad(ops, gemms, xc, dup, wu, ou, layout, ctx.needs_input_grad[3], ctx.needs_input_grad[7])
        elif do_inputs:
            ctx.stash = (dy.clone(), dgate, dup)  # the weight pass follows later
        if not ctx.needs_input_grad[1]:
            dpp = None
        return dxp, dpp, dwg, dwu, dwd, None, None, None, None, None, None, None


def grouped_swiglu(xp: torch.Tensor, pp: torch.Tensor, w_gate: torch.Tensor, w_up: torch.Tensor, w_down: torch.Tensor,
                   layout: MoELayout, out: torch.Tensor | None = None, dx_out: torch.Tensor | None = None,
                   fp8: bool = False, recipe: str = "rowwise") -> torch.Tensor:
    """CUDA bf16 only.  ``w_*`` are ``[E, in, out]``; ``out`` / ``dx_out``: optional ``[>= capacity, hidden]`` buffers the
    block writes its result / its input gradient into (the returned tensor / the gradient then alias them).

    ``fp8=True`` runs the six GEMMs in e4m3 (hidden and intermediate sizes multiples of 16) under ``recipe``:
    ``"rowwise"`` (:class:`_Fp8ExpertGemms`, per-expert row / column scales) or ``"blockwise"``
    (:class:`_BlockwiseFp8ExpertGemms`, DeepSeek-V3's 1x128 / 128x128 scales); :func:`grouped_swiglu_fp8_reference` is
    their PyTorch emulation."""
    _check_fp8_recipe(recipe)
    if fp8:
        bad = [d for d in (*w_gate.shape[1:], w_down.shape[1]) if d % 16]
        if bad:
            raise ValueError(f"grouped_swiglu(fp8=True): hidden and intermediate sizes must be multiples of 16, got {bad}")
    owners, weights = [], []
    for w in (w_gate, w_up, w_down):
        owner = fused_wgrad_owner(w)
        owners.append(owner)
        weights.append(w.detach() if owner is not None else w)
    gemms = _FP8_EXPERT_GEMMS[recipe] if fp8 else _Bf16ExpertGemms
    return _GroupedSwiGLUFunction.apply(xp, pp.float(), *weights, layout, *owners, out, dx_out, gemms)


# ------------------------------------------------------------------------------------------ fp8 emulation
def _scaled(aq, sa, bq, sb) -> torch.Tensor:
    """``(aq @ bq^T) * sa[:, None] * sb[None, :]`` in fp32 (products of e4m3 values are exact in fp32)."""
    return (aq.float() @ bq.float().t()) * sa[:, None] * sb[None, :]


def _blockwise_scaled(aq, sa, bq, sb, dtype) -> torch.Tensor:
    return blockwise_mm_reference(aq, sa, bq, sb, out_dtype=dtype)


# Per recipe, one expert's three GEMMs on bf16 operands: forward (x_e, W[e] [in, out]) -> y_e, dgrad (dy_e, W[e]) -> dx_e,
# wgrad (x_e, dy_e, dtype) -> dW[e].  The blockwise token groups of the weight gradient start at the expert's first row.
_EMULATED_EXPERT_GEMMS = {
    "rowwise": (
        lambda x, w: _scaled(*quantize_rowwise_reference(x), *quantize_colwise_t_reference(w)).to(x.dtype),
        lambda dy, w: _scaled(*quantize_rowwise_reference(dy), *quantize_rowwise_reference(w)).to(dy.dtype),
        lambda x, dy, dt: _scaled(*quantize_colwise_t_reference(x), *quantize_colwise_t_reference(dy)).to(dt),
    ),
    "blockwise": (
        lambda x, w: _blockwise_scaled(*quantize_blockwise_reference(x), *quantize_weight_blocks_reference(w, True), x.dtype),
        lambda dy, w: _blockwise_scaled(*quantize_blockwise_reference(dy), *quantize_weight_blocks_reference(w), dy.dtype),
        lambda x, dy, dt: _blockwise_scaled(*quantize_blockwise_t_reference(x), *quantize_blockwise_t_reference(dy), dt),
    ),
}


class _Fp8GroupedLinearEmulation(Function):
    """``out[rows of e] = x[rows of e] @ W[e]`` with the three GEMMs of the ``recipe``'s expert GEMMs emulated in PyTorch;
    rows outside every expert's range are zero in the output and the input gradient."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, w: torch.Tensor, starts: list[int], counts: list[int], recipe: str = "rowwise"):
        ctx.save_for_backward(x, w)
        ctx.segs = list(zip(starts, counts))
        ctx.gemms = _EMULATED_EXPERT_GEMMS[recipe]
        out = x.new_zeros(x.shape[0], w.shape[2])
        for e, (s0, n) in enumerate(ctx.segs):
            if n > 0:
                out[s0 : s0 + n] = ctx.gemms[0](x[s0 : s0 + n], w[e])
        return out

    @staticmethod
    def backward(ctx: Any, dy: torch.Tensor):  # type: ignore[override]
        x, w = ctx.saved_tensors
        _, dgrad, wgrad = ctx.gemms
        dx = x.new_zeros(x.shape) if ctx.needs_input_grad[0] else None
        dw = torch.zeros(w.shape, dtype=grad_dtype_of(w), device=w.device) if ctx.needs_input_grad[1] else None
        for e, (s0, n) in enumerate(ctx.segs):
            if n == 0:
                continue
            dye = dy[s0 : s0 + n].to(x.dtype)
            if dx is not None:
                dx[s0 : s0 + n] = dgrad(dye, w[e])
            if dw is not None:
                dw[e] = wgrad(x[s0 : s0 + n], dye, dw.dtype)
        return dx, dw, None, None, None


def fp8_grouped_linear_reference(x: torch.Tensor, w: torch.Tensor, starts, counts, recipe: str = "rowwise") -> torch.Tensor:
    """PyTorch emulation of one fp8 grouped projection under ``recipe`` (``"rowwise"`` or ``"blockwise"``); expert ``e``
    owns rows ``[starts[e], starts[e] + counts[e])``."""
    _check_fp8_recipe(recipe)
    return _Fp8GroupedLinearEmulation.apply(x, w, [int(v) for v in starts], [int(v) for v in counts], recipe)


def grouped_swiglu_fp8_reference(xp: torch.Tensor, pp: torch.Tensor, w_gate: torch.Tensor, w_up: torch.Tensor,
                                 w_down: torch.Tensor, starts, counts, recipe: str = "rowwise") -> torch.Tensor:
    """PyTorch emulation of ``grouped_swiglu(..., fp8=True, recipe=recipe)``: the same quantisation of every GEMM operand,
    the SiLU·mul and probability product in fp32, intermediates rounded to the activations' dtype."""
    starts, counts = [int(v) for v in starts], [int(v) for v in counts]
    gate = fp8_grouped_linear_reference(xp, w_gate, starts, counts, recipe)
    up = fp8_grouped_linear_reference(xp, w_up, starts, counts, recipe)
    h = (torch.nn.functional.silu(gate.float()) * up.float() * pp.float()[:, None]).to(xp.dtype)
    return fp8_grouped_linear_reference(h, w_down, starts, counts, recipe)
