"""fp64 references and per-element error bounds for the bandwidth-bound kernels: RMSNorm, SiLU·mul(·probs), RoPE, the
fused q/k RMSNorm + RoPE, the MoE gather-sum and ``sumsq_accumulate``.  Pure torch: works on CPU tensors (self-test) and
CUDA tensors alike.  Every function returns ``(reference, bound)`` pairs computed in fp64 from the exact tensors handed to
the kernel; compare with ``err_ratio`` / ``assert_within`` from ``tests.gemm_reference``.

Bound terms (all kernels compute in fp32):

    u_o                  unit roundoff of the output: 2^-8 bf16, 2^-11 fp16, 2^-24 fp32
    c_n                  max(n / 16, 1) * 2^-22, an fp32 sum of n terms (``ck`` of the GEMM suite)
    U32 = 2^-24          one fp32 rounding
    E_RSQRT = 2^-22      ``rsqrtf`` (MUFU.RSQ) relative error
    e_f(a)               2^-20 + |a| 2^-23: ``1 / (1 + __expf(-a))`` (ex2.approx of a rounded a * log2(e), then a fast
                         reciprocal), relative
"""

from __future__ import annotations

import torch

from tests.gemm_reference import U_BF16, U_F32, ck

U32 = U_F32
U_F16 = 2.0**-11
E_RSQRT = 2.0**-22


def unit_roundoff(dtype: torch.dtype) -> float:
    return {torch.bfloat16: U_BF16, torch.float16: U_F16, torch.float32: U_F32}[dtype]


def rounding(ref: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Bound of rounding ``ref`` to ``dtype``: u_o |ref|, plus half the spacing of fp16's subnormals, or the fp32 flush to
    zero of the fast-math kernels (2^-126)."""
    return unit_roundoff(dtype) * ref.abs() + (2.0**-25 if dtype == torch.float16 else 2.0**-126)


def cn(n: int) -> float:
    return ck(n)


def f32(v: float) -> float:
    """The fp32 value a kernel receives for a Python float argument (eps)."""
    return float(torch.tensor(v, dtype=torch.float32))


def inv_rms_rel(n: int) -> float:
    """Relative bound of an fp32 ``rsqrtf(sum(x^2) / n + eps)``: half the sum's c_n, the divide and add, the rsqrt."""
    return cn(n) / 2 + 2 * E_RSQRT


def _weight(w: torch.Tensor, zero_centered: bool) -> torch.Tensor:
    return w.double() + 1.0 if zero_centered else w.double()


# ----------------------------------------------------------------------------- RMSNorm
def inv_rms_ref(x: torch.Tensor, eps: float) -> tuple[torch.Tensor, torch.Tensor]:
    """x [..., N] -> (1 / sqrt(mean(x^2) + eps) [...], relative bound * |ref|)."""
    ir = torch.rsqrt(x.double().square().mean(-1) + f32(eps))
    return ir, inv_rms_rel(x.shape[-1]) * ir


def rms_norm_fwd_ref(x: torch.Tensor, w: torch.Tensor, eps: float, zero_centered: bool,
                     inv_rms: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """(out, out_bound, inv_rms, inv_rms_bound).  With the kernel's ``inv_rms`` the output is checked against
    ``x * inv_rms * w`` (the normalisation is then checked by the ``inv_rms`` comparison alone); without it the output
    bound also carries the ``inv_rms`` error."""
    ir_ref, ir_bound = inv_rms_ref(x, eps)
    ir = ir_ref if inv_rms is None else inv_rms.double()
    ref = x.double() * ir[..., None] * _weight(w, zero_centered)
    rel = 3 * U32 + (inv_rms_rel(x.shape[-1]) if inv_rms is None else 0.0)
    return ref, rel * ref.abs() + rounding(ref, x.dtype), ir_ref, ir_bound


def _rms_bwd(dy: torch.Tensor, dy_mag: torch.Tensor, dy_rel: float, x: torch.Tensor, ir: torch.Tensor, w: torch.Tensor,
             ir_rel: float, dx_dtype: torch.dtype, dw_dtype: torch.dtype):
    """Shared RMSNorm backward over the last dim.  dy: the incoming gradient in fp64, dy_mag >= |dy| the magnitude its
    fp32 computation carried, dy_rel its relative error (0 for a gradient read from memory); ir [...] fp64; w fp64 [N]."""
    N = x.shape[-1]
    M = x.numel() // max(N, 1)
    ir = ir[..., None]
    xh = x.double() * ir
    g = dy * w
    A = dy_mag * w.abs()
    md = (g * xh).mean(-1, keepdim=True)
    mabs = (A * xh.abs()).mean(-1, keepdim=True)
    dx = ir * (g - xh * md)
    dx_bound = ir * ((4 * U32 + dy_rel) * A + (cn(N) + 8 * U32 + dy_rel) * xh.abs() * mabs
                     + ir_rel * (A + 3 * xh.abs() * mabs)) + 2 * U32 * dx.abs() + rounding(dx, dx_dtype)
    dw = (dy * xh).reshape(-1, N).sum(0)
    S = (dy_mag * xh.abs()).reshape(-1, N).sum(0)
    dw_bound = (cn(M) + 2 * U32 + dy_rel + ir_rel) * S + rounding(dw, dw_dtype)
    return dx, dx_bound, dw, dw_bound


def rms_norm_bwd_ref(dy: torch.Tensor, x: torch.Tensor, w: torch.Tensor, inv_rms: torch.Tensor, zero_centered: bool,
                     ir_rel: float = 0.0):
    """(dx, dx_bound, dw, dw_bound) of ``out = x * inv_rms * w`` with ``inv_rms`` taken as an input (pass the kernel's
    own to check the backward by itself, or the fp64 one with ``ir_rel = inv_rms_rel(N)`` for an end-to-end check)."""
    d = dy.double()
    return _rms_bwd(d, d.abs(), 0.0, x, inv_rms.double(), _weight(w, zero_centered), ir_rel, x.dtype, w.dtype)


# ----------------------------------------------------------------------------- SiLU * mul
def _silu(x: torch.Tensor):
    a = x.double()
    sg = torch.sigmoid(a)
    return a, sg, a * sg, 2.0**-20 + a.abs() * 2.0**-23


def silu_mul_fwd_ref(x: torch.Tensor, y: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """silu(x) * y.  The kernel rounds silu to the storage dtype before the product: one u_o * |silu * y| term for that,
    one for the output."""
    _, _, silu, ef = _silu(x)
    yd = y.double()
    ref = silu * yd
    return ref, rounding(silu, x.dtype) * yd.abs() + (ef + U32) * ref.abs() + rounding(ref, x.dtype)


def silu_mul_bwd_ref(g: torch.Tensor, x: torch.Tensor, y: torch.Tensor):
    """(dx, dx_bound, dy, dy_bound); dx = g * y * sg * (1 + x * (1 - sg)) may cancel, so its bound is absolute in
    |g * y| * (sg + |silu|)."""
    a, sg, silu, ef = _silu(x)
    gd, yd = g.double(), y.double()
    dy = gd * silu
    dx = gd * yd * (sg + silu * (1 - sg))
    return (dx, (ef + 6 * U32) * (gd * yd).abs() * (sg + silu.abs()) + rounding(dx, x.dtype),
            dy, (ef + 2 * U32) * dy.abs() + rounding(dy, x.dtype))


def silu_mul_probs_fwd_ref(x: torch.Tensor, y: torch.Tensor, probs: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """silu(x) * y * probs[:, None] (no intermediate rounding)."""
    _, _, silu, ef = _silu(x)
    ref = silu * y.double() * probs.double()[:, None]
    return ref, (ef + 3 * U32) * ref.abs() + rounding(ref, x.dtype)


def silu_mul_probs_bwd_ref(g: torch.Tensor, x: torch.Tensor, y: torch.Tensor, probs: torch.Tensor):
    """(dx, dx_bound, dy, dy_bound, dprobs, dprobs_bound); dprobs[r] = sum over the cols of g * silu * y, an fp32 sum."""
    a, sg, silu, ef = _silu(x)
    gp = g.double() * probs.double()[:, None]
    yd = y.double()
    dy = gp * silu
    dx = gp * yd * (sg + silu * (1 - sg))
    t = g.double() * silu * yd
    dp = t.sum(-1)
    dp_bound = ((ef + 3 * U32) * t.abs()).sum(-1) + cn(x.shape[-1]) * t.abs().sum(-1)
    return (dx, (ef + 7 * U32) * (gp * yd).abs() * (sg + silu.abs()) + rounding(dx, x.dtype),
            dy, (ef + 3 * U32) * dy.abs() + rounding(dy, x.dtype), dp, dp_bound)


# ----------------------------------------------------------------------------- RoPE
def _rotate(v: torch.Tensor, c: torch.Tensor, s: torch.Tensor, style: int) -> tuple[torch.Tensor, torch.Tensor]:
    """fp64 rotation of the first rope_dim = c.shape[-1] dims of v [..., D] (c, s broadcast against v[..., :rope_dim]).
    HALF (style 0): out = v * c + cat(-v2, v1) * s; INTERLEAVED (1): pairs (2i, 2i+1).  Returns (out, mag) with
    mag = |v * c| + |partner * s| on the rotated dims and 0 on the pass-through dims."""
    rd = c.shape[-1]
    vr = v[..., :rd]
    if style == 0:
        h = rd // 2
        rot = torch.cat([-vr[..., h:], vr[..., :h]], -1)
    else:
        rot = torch.stack([-vr[..., 1::2], vr[..., 0::2]], -1).flatten(-2)
    out = torch.cat([vr * c + rot * s, v[..., rd:]], -1)
    mag = torch.cat([(vr * c).abs() + (rot * s).abs(), torch.zeros_like(v[..., rd:])], -1)
    return out, mag


def rope_ref(x: torch.Tensor, cos_cache: torch.Tensor, sin_cache: torch.Tensor, pos: torch.Tensor, style: int,
             inverse: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """x [T, H, D] bf16 (any token stride); caches [max_pos, rope_dim] fp32; pos [T].  Pass-through dims must be copied
    exactly (bound 0); rotated dims carry two fp32 roundings and the output rounding."""
    c = cos_cache.double()[pos.long()][:, None, :]
    s = sin_cache.double()[pos.long()][:, None, :]
    ref, mag = _rotate(x.double(), c, -s if inverse else s, style)
    bound = (2 * U32 * mag + rounding(ref, x.dtype)) * (mag > 0)
    return ref, bound


# ----------------------------------------------------------------------------- fused q/k RMSNorm + RoPE
def qk_norm_rope_fwd_ref(q: torch.Tensor, k: torch.Tensor, wq: torch.Tensor, wk: torch.Tensor, cos_t: torch.Tensor,
                         sin_t: torch.Tensor, eps: float, zero_centered: bool, style: int,
                         inv_rms: torch.Tensor | None = None):
    """q [T, Hq, D], k [T, Hk, D]; cos_t / sin_t [T, rope_dim] per token.  Returns (q_out, q_bound, k_out, k_bound,
    inv_rms [T, Hq + Hk], inv_rms_bound).  With the kernel's ``inv_rms`` the outputs use it (see ``rms_norm_fwd_ref``)."""
    Hq = q.shape[1]
    D = q.shape[-1]
    ir_ref, ir_bound = inv_rms_ref(torch.cat([q, k], 1), eps)
    ir = ir_ref if inv_rms is None else inv_rms.double()
    rel_ir = inv_rms_rel(D) if inv_rms is None else 0.0
    c, s = cos_t.double()[:, None, :], sin_t.double()[:, None, :]
    outs = []
    for x, w, irx in ((q, wq, ir[:, :Hq]), (k, wk, ir[:, Hq:])):
        y = x.double() * irx[..., None] * _weight(w, zero_centered)
        ref, mag = _rotate(y, c, s, style)
        mag = mag + (mag == 0) * y.abs()  # pass-through dims: the normalised value itself
        outs += [ref, (5 * U32 + rel_ir) * mag + rounding(ref, x.dtype)]
    return (*outs, ir_ref, ir_bound)


def qk_norm_rope_bwd_ref(gq: torch.Tensor, gk: torch.Tensor, q: torch.Tensor, k: torch.Tensor, wq: torch.Tensor,
                         wk: torch.Tensor, cos_t: torch.Tensor, sin_t: torch.Tensor, inv_rms: torch.Tensor,
                         zero_centered: bool, style: int, ir_rel: float = 0.0):
    """(dq, dq_bound, dk, dk_bound, dwq, dwq_bound, dwk, dwk_bound) with ``inv_rms`` [T, Hq + Hk] taken as an input:
    the incoming gradient is rotated back (R(-theta)), then the per-head RMSNorm backward."""
    Hq = q.shape[1]
    c, s = cos_t.double()[:, None, :], sin_t.double()[:, None, :]
    ir = inv_rms.double()
    outs = []
    for g, x, w, irx in ((gq, q, wq, ir[:, :Hq]), (gk, k, wk, ir[:, Hq:])):
        dy, mag = _rotate(g.double(), c, -s, style)
        mag = mag + (mag == 0) * dy.abs()
        outs.append(_rms_bwd(dy, mag, 2 * U32, x, irx, _weight(w, zero_centered), ir_rel, x.dtype, torch.float32))
    (dq, dqb, dwq, dwqb), (dk, dkb, dwk, dwkb) = outs
    return dq, dqb, dk, dkb, dwq, dwqb, dwk, dwkb


# ----------------------------------------------------------------------------- MoE gather-sum, sumsq
def moe_gather_ref(yp: torch.Tensor, row_map: torch.Tensor, T: int, k: int, dpp: torch.Tensor | None = None):
    """y[t] = sum_j yp[row_map[t, j]] over the kept rows (row_map >= 0): a sum of k terms in fp32, rounded to bf16.
    Returns (y, y_bound, dprobs) with dprobs[t, j] = dpp[row_map[t, j]] or 0 (exact)."""
    rm = row_map.long().reshape(T, k)
    keep = rm >= 0
    rows = yp.double()[rm.clamp_min(0)] * keep[..., None]  # [T, k, H]
    y = rows.sum(1)
    bound = cn(k) * rows.abs().sum(1) + rounding(y, yp.dtype)
    dprobs = None
    if dpp is not None:
        dprobs = torch.where(keep, dpp.double()[rm.clamp_min(0)], torch.zeros((), dtype=torch.float64, device=yp.device))
    return y, bound, dprobs


def sumsq_ref(x: torch.Tensor, out0: float, adds: int = 1) -> tuple[float, float]:
    """``out += sum(x^2)``: the contract is an accumulate.  The kernel sums in fp32 per block and adds each block's sum to
    ``out`` atomically (``adds`` rounded additions to a running total of at most |out0| + sum(x^2))."""
    ss = float(x.double().square().sum())
    return out0 + ss, cn(x.numel()) * ss + adds * U32 * (abs(out0) + ss)
