"""FP8 (e4m3) linear algebra on the Hopper tensor cores (wgmma).

Three operand recipes.  The tensor core sums an MMA chain in a reduced-precision accumulator (not fp32), so how long the
chains are sets the accuracy of a long reduction:

* **row / column scaling**: one fp32 scale per row of each operand (per token / per output channel), applied to the
  accumulator in the GEMM epilogue; the whole of K is one chain (no promotion).  The default recipe of
  :class:`Fp8LinearFunction` for all three GEMMs of a linear layer (forward, input gradient, weight gradient); the two
  backward GEMMs need K-major operands along the *other* dimension, which the transposing column-wise quantiser produces
  in one pass.
* **MXFP8**: OCP micro-scaling - one power-of-two (UE8M0) scale per 32 consecutive
  K-elements; every K=32 wgmma produces a partial product that is added to an fp32 accumulator with its two scales.
* **blockwise** (DeepSeek-V3): one fp32 scale per 1x128 group of an activation row and per 128x128 block of a weight,
  both along the reduction dimension.  Every 128-deep k-block of the GEMM is summed by the tensor core into a fresh
  accumulator and added to the fp32 accumulator with its row x column scale ("promotion"), so one outlier only sets the
  scale of its own group and the accumulation is never one long reduced-precision chain.  Scales are stored
  k-block-major, ``[ceil(K/128), rows]``.  In the linear layer (``recipe="blockwise"``) the weight gradient is written
  by the GEMM in the gradient dtype (fp32 or bf16).

The reference framework has no fp8 path of its own (its published fp8 numbers come from torchao-style recipes layered on
top); this module is the native equivalent.  Every function has a PyTorch emulation (same rounding, same scale rules) that
runs on CPU and is the numerical oracle of the GPU tests.
"""

from __future__ import annotations

from typing import Any, Callable, NamedTuple

import torch
from torch import nn
from torch.autograd import Function

from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection

from .._native import grad_dtype_of, native_ops, on_gpu

E4M3_MAX = 448.0
FP8 = torch.float8_e4m3fn


# ---------------------------------------------------------------------------------------------------- emulation
def quantize_rowwise_reference(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    xf = x.float()
    scale = _group_scales(xf.abs().amax(dim=1))
    q = (xf / scale[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(FP8)
    return q, scale


def quantize_colwise_t_reference(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    q, scale = quantize_rowwise_reference(x.t())
    return q, scale


def quantize_colwise_t_batched_reference(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [E, R, C]`` -> ``(qT [E, C, R], scale [E, C])``: the transposing quantiser applied to every ``x[e]``."""
    parts = [quantize_colwise_t_reference(xe) for xe in x]
    return torch.stack([q for q, _ in parts]), torch.stack([s for _, s in parts])


def quantize_segments_t_reference(x: torch.Tensor, starts, counts) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [R, C]`` with expert ``e`` on rows ``[starts[e], starts[e] + counts[e])`` -> ``(qT [C, R], scale [E, C])``: one
    scale per (expert, column) over the expert's rows (1 for an expert without rows or with all-zero values); every row of
    ``x`` outside the experts' ranges comes out as zero in ``qT``."""
    starts, counts = [int(v) for v in starts], [int(v) for v in counts]
    qt = torch.zeros(x.shape[1], x.shape[0], dtype=FP8, device=x.device)
    scale = torch.ones(len(counts), x.shape[1], dtype=torch.float32, device=x.device)
    for e, (s0, n) in enumerate(zip(starts, counts)):
        if n > 0:
            qt[:, s0 : s0 + n], scale[e] = quantize_colwise_t_reference(x[s0 : s0 + n])
    return qt, scale


def mx_scale_exponent(amax: torch.Tensor) -> torch.Tensor:
    """Smallest integer ``e`` with ``amax / 2**e <= 448`` (``-127`` for all-zero groups), clamped to [-126, 126]."""
    # 448 = 1.75 * 2**8: with amax = m * 2**x (1 <= m < 2) the answer is x - 8 (+1 if m > 1.75) - exact, no logarithms
    frac, exp = torch.frexp(amax.float().clamp_min(torch.finfo(torch.float32).tiny))  # amax = frac * 2**exp, frac in [0.5, 1)
    e = (exp - 1 - 8 + (frac * 2 > 1.75).to(exp.dtype)).clamp(-126, 126).float()
    return torch.where(amax > 0, e, torch.full_like(e, -127)).to(torch.int32)


def quantize_mx_reference(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Returns ``(q[M,K] e4m3, e[M, K/32] int32)``: ``x ~= q * 2**e`` per 32-element group (the native op packs ``e + 127``
    into the tensor-core block layout instead, see :func:`unpack_mx_scales`)."""
    M, K = x.shape
    g = x.float().view(M, K // 32, 32)
    e = mx_scale_exponent(g.abs().amax(dim=-1))
    inv = torch.where(e == -127, torch.zeros_like(e, dtype=torch.float32), torch.exp2(-e.float()))
    q = (g * inv[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(FP8).view(M, K)
    return q, e


def unpack_mx_scales(sf: torch.Tensor, rows: int, K: int) -> torch.Tensor:
    """Block layout ``[row_blocks, K/128, 512]`` (byte ``(r%32)*16 + (r//32)*4 + g``) -> exponents ``[rows, K/32]``."""
    nb, kb, _ = sf.shape
    t = sf.view(nb, kb, 32, 4, 4).permute(0, 3, 2, 1, 4)  # [blk, r//32, r%32, kblock, g]
    return (t.reshape(nb * 128, kb * 4)[:rows].to(torch.int32) - 127)


def dequantize_mx(q: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    M, K = q.shape
    return (q.float().view(M, K // 32, 32) * torch.exp2(e.float())[..., None]).view(M, K)


def _scaled_mm_reference(aq, sa, bq, sb) -> torch.Tensor:
    return ((aq.float() @ bq.float().t()) * sa[:, None] * sb[None, :]).to(torch.bfloat16)


def _group_scales(amax: torch.Tensor) -> torch.Tensor:
    """``amax / 448``, at least 2**-126 (the smallest normal fp32, so that the kernels' reciprocal stays finite under
    flush-to-zero), and 1 for an all-zero group."""
    return torch.where(amax > 0, (amax / E4M3_MAX).clamp_min(2.0**-126), torch.ones_like(amax))


def quantize_blockwise_reference(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [M, K]`` -> ``(q [M, K] e4m3, s [ceil(K/128), M] fp32)`` with ``x[m, k] ~= q[m, k] * s[k // 128, m]``: one scale
    per 1x128 group of every row (a partial last group covers its valid elements; an all-zero group gets scale 1)."""
    M, K = x.shape
    G = (K + 127) // 128
    xg = torch.nn.functional.pad(x.float(), (0, G * 128 - K)).view(M, G, 128)
    scale = _group_scales(xg.abs().amax(dim=-1))  # [M, G]
    q = (xg / scale[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(FP8).view(M, G * 128)[:, :K]
    return q.contiguous(), scale.t().contiguous()


def quantize_blockwise_t_reference(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [M, C]`` -> ``(qT [C, M], s [ceil(M/128), C])``: the transposed copy with one scale per 128 rows (tokens) of every
    column (channel)."""
    return quantize_blockwise_reference(x.t())


def quantize_weight_blocks_reference(w: torch.Tensor, transpose: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
    """``w [N, K]`` -> one scale per 128x128 block, repeated on each row of the copy the GEMM reads:
    ``(q [N, K], s [ceil(K/128), N])``, or with ``transpose`` ``(qT [K, N], s [ceil(N/128), K])``.  ``qT`` is bitwise ``q^T``."""
    N, K = w.shape
    Nb, Kb = (N + 127) // 128, (K + 127) // 128
    wb = torch.nn.functional.pad(w.float(), (0, Kb * 128 - K, 0, Nb * 128 - N)).view(Nb, 128, Kb, 128)
    scale = _group_scales(wb.abs().amax(dim=(1, 3)))  # [Nb, Kb]
    q = (wb / scale[:, None, :, None]).clamp(-E4M3_MAX, E4M3_MAX).to(FP8).view(Nb * 128, Kb * 128)[:N, :K]
    if transpose:
        return q.t().contiguous(), scale.repeat_interleave(128, dim=1)[:, :K].contiguous()
    return q.contiguous(), scale.t().repeat_interleave(128, dim=1)[:, :N].contiguous()


def quantize_expert_weight_blocks_reference(w: torch.Tensor, transpose: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """``w [E, in, out]`` -> :func:`quantize_weight_blocks_reference` of every ``w[e]``: with ``transpose`` (the grouped
    forward) ``(qT [E, out, in], s [E, ceil(in/128), out])``, else (the input gradient) ``(q [E, in, out], s [E, ceil(out/128), in])``."""
    parts = [quantize_weight_blocks_reference(we, transpose) for we in w]
    return torch.stack([q for q, _ in parts]), torch.stack([s for _, s in parts])


def _segment_rows(x: torch.Tensor, starts, counts) -> torch.Tensor:
    """``x`` with every row outside the experts' ranges ``[starts[e], starts[e] + counts[e])`` set to zero."""
    keep = torch.zeros(x.shape[0], dtype=torch.bool, device=x.device)
    for s0, n in zip(starts, counts):
        keep[int(s0) : int(s0) + int(n)] = True
    return torch.where(keep[:, None], x, torch.zeros((), dtype=x.dtype, device=x.device))


def quantize_blockwise_segments_reference(x: torch.Tensor, starts, counts) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [cap, C]`` in the MoE layout -> ``(q [cap, C], s [ceil(C/128), cap])``: 1x128 row groups of the experts' rows;
    every other row quantises to zero codes with scale 1."""
    return quantize_blockwise_reference(_segment_rows(x, starts, counts))


def quantize_blockwise_segments_t_reference(x: torch.Tensor, starts, counts) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [cap, C]`` in the MoE layout (segments start on 128-row boundaries) -> ``(qT [C, cap], s [cap/128, C])``: one scale
    per 128-token group of every channel, the groups of expert ``e`` starting at its first row and ending at its last;
    every row outside the experts' ranges quantises to zero (scale 1 for a group without rows)."""
    return quantize_blockwise_t_reference(_segment_rows(x, starts, counts))


def blockwise_mm_reference(aq, sa, bq, sb, out_dtype: torch.dtype = torch.bfloat16, acc_dtype: torch.dtype = torch.float32):
    """``sum_kb (aq[:, kb] @ bq[:, kb]^T) * sa[kb, :, None] * sb[kb, None, :]`` over the 128-deep k-blocks ``kb``."""
    K = aq.shape[1]
    acc = torch.zeros(aq.shape[0], bq.shape[0], dtype=acc_dtype, device=aq.device)
    for kb in range((K + 127) // 128):
        ks = slice(kb * 128, min(K, kb * 128 + 128))
        part = aq[:, ks].to(acc_dtype) @ bq[:, ks].to(acc_dtype).t()
        acc += part * sa[kb].to(acc_dtype)[:, None] * sb[kb].to(acc_dtype)[None, :]
    return acc.to(out_dtype)


# ---------------------------------------------------------------------------------------------------- public ops
def quantize_rowwise(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    return native_ops().quantize_rowwise(x) if on_gpu(x) else quantize_rowwise_reference(x)


def quantize_colwise_t(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    return native_ops().quantize_colwise_t(x) if on_gpu(x) else quantize_colwise_t_reference(x)


def scaled_mm(aq: torch.Tensor, sa: torch.Tensor, bq: torch.Tensor, sb: torch.Tensor) -> torch.Tensor:
    """``(aq @ bq^T) * sa[:, None] * sb[None, :]`` -> bf16."""
    if on_gpu(aq):
        out = torch.empty(aq.shape[0], bq.shape[0], device=aq.device, dtype=torch.bfloat16)
        native_ops().gemm_fp8(aq, bq, sa, sb, 1.0, out)
        return out
    return _scaled_mm_reference(aq, sa, bq, sb)


def mx_mm(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """``a[M,K] @ b[N,K]^T`` with both operands quantised to MXFP8 on the fly -> bf16."""
    if on_gpu(a):
        ops = native_ops()
        aq, sfa = ops.quantize_mx(a)
        bq, sfb = ops.quantize_mx(b)
        out = torch.empty(a.shape[0], b.shape[0], device=a.device, dtype=torch.bfloat16)
        ops.gemm_mxfp8(aq, sfa, bq, sfb, out)
        return out
    aq, ea = quantize_mx_reference(a)
    bq, eb = quantize_mx_reference(b)
    return (dequantize_mx(aq, ea) @ dequantize_mx(bq, eb).t()).to(torch.bfloat16)


def quantize_blockwise(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [M, K]`` -> ``(q [M, K], s [ceil(K/128), M])``: 1x128 groups along the reduction dimension."""
    return native_ops().quantize_blockwise(x) if on_gpu(x) else quantize_blockwise_reference(x)


def quantize_blockwise_t(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """``x [M, C]`` -> ``(qT [C, M], s [ceil(M/128), C])``: 128-token groups of every channel, transposed copy."""
    return native_ops().quantize_blockwise_t(x) if on_gpu(x) else quantize_blockwise_t_reference(x)


def quantize_weight_blocks(w: torch.Tensor, transpose: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
    """``w [N, K]`` -> 128x128-block scaled ``(q [N, K], s [ceil(K/128), N])`` or ``(qT [K, N], s [ceil(N/128), K])``."""
    return native_ops().quantize_weight_blocks(w, transpose) if on_gpu(w) else quantize_weight_blocks_reference(w, transpose)


def blockwise_mm(aq: torch.Tensor, sa: torch.Tensor, bq: torch.Tensor, sb: torch.Tensor, out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``sum_kb (aq[:, kb] @ bq[:, kb]^T) * sa[kb, :, None] * sb[kb, None, :]`` -> ``out_dtype`` (bf16 or fp32), with the
    per-(k-block, row) scales of :func:`quantize_blockwise`, :func:`quantize_blockwise_t` and :func:`quantize_weight_blocks`."""
    if on_gpu(aq):
        out = torch.empty(aq.shape[0], bq.shape[0], device=aq.device, dtype=out_dtype)
        native_ops().gemm_fp8_blockwise(aq, sa, bq, sb, out)
        return out
    return blockwise_mm_reference(aq, sa, bq, sb, out_dtype)


class _Recipe(NamedTuple):
    """One fp8 recipe of the dense linear layer: its size rule and its three GEMMs."""

    granule: int  # the feature sizes must be multiples of it
    tokens_too: bool  # ... and so must the token count
    forward: Callable[[torch.Tensor, torch.Tensor], torch.Tensor]  # (x2, w) -> y2
    dgrad: Callable[[torch.Tensor, torch.Tensor], torch.Tensor]  # (dy, w) -> dx2
    wgrad: Callable[[torch.Tensor, torch.Tensor, torch.dtype], torch.Tensor]  # (dy, x2, grad_dtype) -> dW


# row / column scaling:
#   forward  y  = Q_row(x)  · Q_row(W)^T        scales: token x output channel
#   dgrad    dx = Q_row(dy) · Q_colT(W)^T       Q_colT(W) = W^T stored [in, out], scale per input channel
#   wgrad    dW = Q_colT(dy) · Q_colT(x)^T      both transposed copies come from the transposing quantiser
def _rowwise_forward(x2, w):
    xq, sx = quantize_rowwise(x2)
    wq, sw = quantize_rowwise(w)
    return scaled_mm(xq, sx, wq, sw)


def _rowwise_dgrad(dy, w):
    dyq, sdy = quantize_rowwise(dy)
    wtq, swt = quantize_colwise_t(w)  # [in, out]
    return scaled_mm(dyq, sdy, wtq, swt)


def _rowwise_wgrad(dy, x2, grad_dtype):
    dytq, sdyt = quantize_colwise_t(dy)  # [out, tokens]
    xtq, sxt = quantize_colwise_t(x2)  # [in, tokens]
    return scaled_mm(dytq, sdyt, xtq, sxt).to(grad_dtype)


# MXFP8 (e4m3 elements, one power-of-two scale per 32 elements of the reduction dimension, applied to the K=32 partial
# products of the GEMM).  Every GEMM quantises both operands along its own reduction dimension, so the backward GEMMs work
# on transposed copies:
#   forward  y  = MX(x)[M,K]    · MX(W)[N,K]^T          reduction over in
#   dgrad    dx = MX(dy)[M,N]   · MX(W^T)[K,N]^T        reduction over out
#   wgrad    dW = MX(dy^T)[N,M] · MX(x^T)[K,M]^T        reduction over tokens
# in, out and the token count must be multiples of 128 (one scale-factor block of the tensor core).
def _mx_dgrad(dy, w):
    return mx_mm(dy, w.t().contiguous())


def _mx_wgrad(dy, x2, grad_dtype):
    return mx_mm(dy.t().contiguous(), x2.t().contiguous()).to(grad_dtype)


# DeepSeek-V3's blockwise scaling with promoted accumulation:
#   forward  y  = Q_blk(x)  · Q_W(W)^T           x: 1x128 groups along in; W: 128x128 blocks
#   dgrad    dx = Q_blk(dy) · Q_W(W^T)^T         dy: 1x128 groups along out; the transposed copy of W's blocks
#   wgrad    dW = Q_blkT(dy) · Q_blkT(x)^T       128-token groups of every channel, written in the gradient dtype
# Feature sizes must be multiples of 16; the token count is free.
def _blockwise_forward(x2, w):
    xq, sx = quantize_blockwise(x2)
    wq, sw = quantize_weight_blocks(w)
    return blockwise_mm(xq, sx, wq, sw)


def _blockwise_dgrad(dy, w):
    dyq, sdy = quantize_blockwise(dy)
    wtq, swt = quantize_weight_blocks(w, transpose=True)  # [in, out]
    return blockwise_mm(dyq, sdy, wtq, swt)


def _blockwise_wgrad(dy, x2, grad_dtype):
    dytq, sdyt = quantize_blockwise_t(dy)  # [out, tokens]
    xtq, sxt = quantize_blockwise_t(x2)  # [in, tokens]
    return blockwise_mm(dytq, sdyt, xtq, sxt, out_dtype=grad_dtype)


_LINEAR_RECIPES = {
    "rowwise": _Recipe(16, False, _rowwise_forward, _rowwise_dgrad, _rowwise_wgrad),
    "mx": _Recipe(128, True, mx_mm, _mx_dgrad, _mx_wgrad),
    "blockwise": _Recipe(16, False, _blockwise_forward, _blockwise_dgrad, _blockwise_wgrad),
}


def _linear_recipe(recipe: str) -> _Recipe:
    if recipe not in _LINEAR_RECIPES:
        raise ValueError(f"unknown fp8 recipe {recipe!r}")
    return _LINEAR_RECIPES[recipe]


class Fp8LinearFunction(Function):
    """``y = x @ W^T`` with all three GEMMs (forward, input gradient, weight gradient) in e4m3, bf16 in / out, under
    ``recipe`` (default ``"rowwise"``).  Nothing quantised is kept between forward and backward: the backward quantises
    again from the saved bf16 ``x`` and ``W``."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, weight: torch.Tensor, recipe: str = "rowwise") -> torch.Tensor:
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        ctx.recipe = _linear_recipe(recipe)
        ctx.save_for_backward(x2, weight)
        ctx.x_shape = x.shape
        return ctx.recipe.forward(x2, weight).view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx: Any, grad_output: torch.Tensor):  # type: ignore[override]
        x2, weight = ctx.saved_tensors
        dy = grad_output.reshape(-1, grad_output.shape[-1])
        if not dy.is_contiguous():
            dy = dy.contiguous()
        dx = dw = None
        if ctx.needs_input_grad[0] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.inputs):
            dx = ctx.recipe.dgrad(dy, weight).view(ctx.x_shape)
        if ctx.needs_input_grad[1] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.weight):
            dw = ctx.recipe.wgrad(dy, x2, grad_dtype_of(weight))
        return dx, dw, None


def fp8_linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None = None, recipe: str = "rowwise") -> torch.Tensor:
    """``x @ weight^T (+ bias)`` in fp8 (:class:`Fp8LinearFunction`).  ``recipe="rowwise"``: dynamic per-row / per-column
    fp32 scales (feature sizes multiples of 16); ``recipe="mx"``: MXFP8 block scaling (feature sizes and token count
    multiples of 128); ``recipe="blockwise"``: DeepSeek-V3's 1x128 / 128x128 scaling with promoted accumulation (feature
    sizes multiples of 16, any token count)."""
    r = _linear_recipe(recipe)
    granule = r.granule
    tokens = x.numel() // max(x.shape[-1], 1)
    if x.shape[-1] % granule or weight.shape[0] % granule or (r.tokens_too and tokens % granule):
        raise ValueError(f"fp8_linear[{recipe}]: sizes must be multiples of {granule} (got in={x.shape[-1]}, out={weight.shape[0]}, "
                         f"tokens={tokens})")
    if on_gpu(x) and (x.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16):
        raise RuntimeError("fp8_linear: bf16 activations and weights required on CUDA")
    out = Fp8LinearFunction.apply(x, weight, recipe)
    return out if bias is None else out + bias


class Fp8Linear(nn.Linear):
    """Drop-in ``nn.Linear`` whose matmuls run in e4m3 (weights stay bf16 master copies); ``fp8_recipe`` (class default
    ``"rowwise"``, set per instance by :func:`convert_linears_to_fp8`) selects the scaling scheme."""

    fp8_recipe: str = "rowwise"

    def forward(self, x: torch.Tensor) -> torch.Tensor:  # type: ignore[override]
        return fp8_linear(x, self.weight, self.bias, recipe=self.fp8_recipe)


def convert_linears_to_fp8(module: nn.Module, predicate=lambda name, m: True, recipe: str = "rowwise") -> int:
    """Re-classes every eligible linear layer of ``module`` to :class:`Fp8Linear` in place: plain ``nn.Linear`` and the
    framework's ``module.block.linear.Linear`` (not LoRA wrappers or other subclasses), feature dims multiples of 16 (128 for
    the ``"mx"`` recipe), ``predicate(name, module)`` true.  Parameters are shared, state-dict keys unchanged.  Returns the
    number converted."""
    from d9d_b200.module.block.linear import Linear as NativeLinear

    granule = _linear_recipe(recipe).granule
    n = 0
    for name, m in module.named_modules():
        if type(m) in (nn.Linear, NativeLinear) and m.in_features % granule == 0 and m.out_features % granule == 0 and predicate(name, m):
            m.__class__ = Fp8Linear
            m.fp8_recipe = recipe
            n += 1
    return n


__all__ = [
    "Fp8Linear", "Fp8LinearFunction", "blockwise_mm", "blockwise_mm_reference",
    "convert_linears_to_fp8", "dequantize_mx", "fp8_linear", "mx_mm", "mx_scale_exponent",
    "quantize_blockwise", "quantize_blockwise_reference", "quantize_blockwise_segments_reference",
    "quantize_blockwise_segments_t_reference", "quantize_blockwise_t", "quantize_blockwise_t_reference",
    "quantize_expert_weight_blocks_reference",
    "quantize_colwise_t", "quantize_colwise_t_batched_reference", "quantize_colwise_t_reference", "quantize_mx_reference",
    "quantize_segments_t_reference", "quantize_rowwise", "quantize_rowwise_reference", "quantize_weight_blocks",
    "quantize_weight_blocks_reference", "scaled_mm", "unpack_mx_scales",
]
