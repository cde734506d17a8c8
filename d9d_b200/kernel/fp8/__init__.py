"""FP8 (e4m3) linear algebra on the Hopper tensor cores (wgmma).

Two operand recipes, both with fp32 accumulation in registers and a bf16 result:

* **row / column scaling**: one fp32 scale per row of each operand (per token / per output channel),
  applied to the accumulator in the GEMM epilogue.  Used by :class:`Fp8LinearFunction` for all three GEMMs of a linear
  layer (forward, input gradient, weight gradient); the two backward GEMMs need K-major operands along the *other*
  dimension, which the transposing column-wise quantiser produces in one pass.
* **MXFP8**: OCP micro-scaling - one power-of-two (UE8M0) scale per 32 consecutive
  K-elements; every K=32 wgmma produces a partial product that is added to the accumulator with its two scales.

The reference framework has no fp8 path of its own (its published fp8 numbers come from torchao-style recipes layered on
top); this module is the native equivalent.  Every function has a PyTorch emulation (same rounding, same scale rules) that
runs on CPU and is the numerical oracle of the GPU tests.
"""

from __future__ import annotations

from typing import Any

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
    amax = xf.abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
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


class Fp8LinearFunction(Function):
    """``y = x @ W^T`` with all three GEMMs in e4m3 (dynamic row / column scaling, bf16 in / out).

    forward  ``y  = Q_row(x)  · Q_row(W)^T``        scales: token x output channel
    dgrad    ``dx = Q_row(dy) · Q_colT(W)^T``       ``Q_colT(W)`` = ``W^T`` stored [in, out], scale per input channel
    wgrad    ``dW = Q_colT(dy) · Q_colT(x)^T``      both transposed copies come from the transposing quantiser
    """

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        xq, sx = quantize_rowwise(x2)
        wq, sw = quantize_rowwise(weight)
        ctx.save_for_backward(x2, weight)
        ctx.x_shape = x.shape
        return scaled_mm(xq, sx, wq, sw).view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx: Any, grad_output: torch.Tensor):  # type: ignore[override]
        x2, weight = ctx.saved_tensors
        dy = grad_output.reshape(-1, grad_output.shape[-1])
        if not dy.is_contiguous():
            dy = dy.contiguous()
        dx = dw = None
        if ctx.needs_input_grad[0] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.inputs):
            dyq, sdy = quantize_rowwise(dy)
            wtq, swt = quantize_colwise_t(weight)  # [in, out]
            dx = scaled_mm(dyq, sdy, wtq, swt).view(ctx.x_shape)
        if ctx.needs_input_grad[1] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.weight):
            dytq, sdyt = quantize_colwise_t(dy)  # [out, tokens]
            xtq, sxt = quantize_colwise_t(x2)  # [in, tokens]
            dw = scaled_mm(dytq, sdyt, xtq, sxt).to(grad_dtype_of(weight))
        return dx, dw


class MxFp8LinearFunction(Function):
    """``y = x @ W^T`` with all three GEMMs in **MXFP8** (e4m3 elements, one power-of-two scale per 32 elements of the
    reduction dimension, applied to the K=32 partial products of the GEMM).

    Every GEMM quantises both operands along *its own* reduction dimension, so the backward GEMMs work on transposed copies:

    forward  ``y  = MX(x)[M,K]    · MX(W)[N,K]^T``          reduction over ``in``
    dgrad    ``dx = MX(dy)[M,N]   · MX(W^T)[K,N]^T``        reduction over ``out``
    wgrad    ``dW = MX(dy^T)[N,M] · MX(x^T)[K,M]^T``        reduction over tokens

    ``in``, ``out`` and the token count must be multiples of 128 (one scale-factor block of the tensor core).
    """

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        ctx.save_for_backward(x2, weight)
        ctx.x_shape = x.shape
        return mx_mm(x2, weight).view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx: Any, grad_output: torch.Tensor):  # type: ignore[override]
        x2, weight = ctx.saved_tensors
        dy = grad_output.reshape(-1, grad_output.shape[-1])
        if not dy.is_contiguous():
            dy = dy.contiguous()
        dx = dw = None
        if ctx.needs_input_grad[0] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.inputs):
            dx = mx_mm(dy, weight.t().contiguous()).view(ctx.x_shape)
        if ctx.needs_input_grad[1] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.weight):
            dw = mx_mm(dy.t().contiguous(), x2.t().contiguous()).to(grad_dtype_of(weight))
        return dx, dw


def fp8_linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None = None, recipe: str = "rowwise") -> torch.Tensor:
    """``x @ weight^T (+ bias)`` in fp8.  ``recipe="rowwise"``: dynamic per-row / per-column fp32 scales
    (:class:`Fp8LinearFunction`, feature sizes multiples of 16); ``recipe="mx"``: MXFP8 block scaling
    (:class:`MxFp8LinearFunction`, feature sizes and token count multiples of 128)."""
    if recipe not in ("rowwise", "mx"):
        raise ValueError(f"unknown fp8 recipe {recipe!r}")
    granule = 16 if recipe == "rowwise" else 128
    tokens = x.numel() // max(x.shape[-1], 1)
    if x.shape[-1] % granule or weight.shape[0] % granule or (recipe == "mx" and tokens % granule):
        raise ValueError(f"fp8_linear[{recipe}]: sizes must be multiples of {granule} (got in={x.shape[-1]}, out={weight.shape[0]}, "
                         f"tokens={tokens})")
    if on_gpu(x) and (x.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16):
        raise RuntimeError("fp8_linear: bf16 activations and weights required on CUDA")
    out = (Fp8LinearFunction if recipe == "rowwise" else MxFp8LinearFunction).apply(x, weight)
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

    if recipe not in ("rowwise", "mx"):
        raise ValueError(f"unknown fp8 recipe {recipe!r}")
    granule = 16 if recipe == "rowwise" else 128
    n = 0
    for name, m in module.named_modules():
        if type(m) in (nn.Linear, NativeLinear) and m.in_features % granule == 0 and m.out_features % granule == 0 and predicate(name, m):
            m.__class__ = Fp8Linear
            m.fp8_recipe = recipe
            n += 1
    return n


__all__ = [
    "Fp8Linear", "Fp8LinearFunction", "MxFp8LinearFunction", "convert_linears_to_fp8", "dequantize_mx", "fp8_linear", "mx_mm", "mx_scale_exponent",
    "quantize_colwise_t", "quantize_colwise_t_batched_reference", "quantize_colwise_t_reference", "quantize_mx_reference",
    "quantize_segments_t_reference", "quantize_rowwise", "quantize_rowwise_reference",
    "scaled_mm", "unpack_mx_scales",
]
