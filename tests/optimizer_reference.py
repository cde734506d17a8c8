"""Exact model of the stochastic-rounding kernels' random streams, an fp64 AdamW reference with a per-element bound, and the
checker that compares a kernel's stochastically rounded bf16 output with both.  Pure torch: works on CPU tensors
(self-test) and CUDA tensors alike.

Random stream.  ``philox4x32`` (``ops/csrc/common.cuh``) is Philox4x32-10 as published with Random123: the 64-bit
counter is the words (c0, c1) = (low, high) with c2 = c3 = 0, the 64-bit key is (k0, k1) = (low, high).  Each draw gives
four 32-bit words, i.e. eight 16-bit halves, one per element of an 8-element vector: element ``e`` of a stream uses
counter ``e >> 3``, word ``(e & 7) >> 1`` and the low half when ``e`` is even, the high half when it is odd.  The stream
position ``e`` is

    sr_copy_                   the element index
    adamw_sr_multi_            rng_base + element index (rng_base is a multiple of 8, so the vector of 8 never straddles
                               two counters); keys seed, seed + 42, seed + 67 (64-bit sums) for p, exp_avg, exp_avg_sq
    nvl_adamw_shard_           the element's global arena index, whatever the shard; the same three keys

Rounding.  ``sr_bf16_bits`` adds the 16 random bits to the fp32 bit pattern and keeps the high half, so a value between
two bf16 neighbours rounds up with probability equal to its distance from the lower one: ``(bits + r) >> 16``.  An inf
stays the same inf and a NaN stays a NaN.

Bound.  The kernels compute AdamW in fp32 in this order (``adamw_sr_kernel``, ``nvl_adamw_shard_kernel``):

    g  = g_in * gs                      pw = p * (1 - lr * wd)
    m' = b1 * m + (1 - b1) * g          v' = b2 * v + (1 - b2) * (g * g)
    pw -= (lr * (m' / bc1)) / (sqrtf(v' / bc2) + eps)

``adamw_ref`` computes the same expression in fp64 from the exact inputs and the fp32 scalars the kernel receives
(``bc1, bc2 = float32(1 - beta^step)``), and a first-order absolute bound on the kernel's fp32 value built from these terms:

    U32 = 2^-24      one fp32 rounding (add, multiply: round to nearest)
    E_DIV = 2^-22    ``/`` under ``--use_fast_math`` is ``div.approx.ftz.f32``: at most 2 ulp for divisors in
                     [2^-126, 2^126] (PTX ISA, ``div``); 2 ulp <= 2^-22 relative
    E_SQRT = 2^-22   ``sqrtf`` under ``--use_fast_math`` is ``sqrt.approx.ftz.f32`` (PTX ISA, ``sqrt``: relative error
                     2^-23); taken as 2 ulp, like the division
    FTZ = 2^-126     ``.ftz``: an operation whose result would be subnormal returns zero

The moments are bounded over their terms, not their result, so that cancellation is covered:
``|m' - ref| <= 4 U32 (|b1 m| + |(1 - b1) g|)`` (the product b1 m, the 1 - b1, the scaled gradient, the product and the
sum), ``|v' - ref| <= 6 U32 (|b2 v| + |(1 - b2) g^2|)`` (the square adds two).  The bias corrections, the square root,
``+ eps``, ``lr *`` and the final division carry their errors through to the update, and the parameter's bound is taken
over ``|p (1 - lr wd)| + |update|``.  Every step also adds one FTZ.  A factor 1 + 2^-20 covers the second-order terms.
"""

from __future__ import annotations

import math

import torch

from tests.gemm_reference import U_F32, assert_within

U32 = U_F32
E_DIV = 2.0**-22
E_SQRT = 2.0**-22
FTZ = 2.0**-126
SECOND_ORDER = 1.0 + 2.0**-20
MAX_AMBIGUOUS = 2.0**-8
MASK32 = 0xFFFFFFFF
MASK64 = (1 << 64) - 1
M_STATE, V_STATE = 42, 67  # key offsets of the exp_avg and exp_avg_sq streams


def f32(v: float) -> float:
    """The fp32 value a kernel receives for a Python float argument."""
    return float(torch.tensor(v, dtype=torch.float32))


# ----------------------------------------------------------------------------- Philox4x32-10
_PHILOX_M = (0xD2511F53, 0xCD9E8D57)
_PHILOX_W = (0x9E3779B9, 0xBB67AE85)


def _mulhilo(m: int, c: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(hi, lo) 32-bit words of m * c for 32-bit c held in int64, without overflowing int64: m = mh 2^16 + ml."""
    a = c * (m & 0xFFFF)
    b = c * (m >> 16)
    lo = (((b & 0xFFFF) << 16) + a) & MASK32
    hi = (b + (a >> 16)) >> 16
    return hi, lo


def philox4x32_10(c0, c1, c2, c3, k0: int, k1: int) -> torch.Tensor:
    """Philox4x32-10 of the counter words (int64 tensors or ints holding 32-bit values) and key words; returns [..., 4]."""
    dev = next((x.device for x in (c0, c1, c2, c3) if isinstance(x, torch.Tensor)), None)
    c = [torch.as_tensor(x, dtype=torch.int64, device=dev) for x in (c0, c1, c2, c3)]
    c = list(torch.broadcast_tensors(*c))
    for _ in range(10):
        hi0, lo0 = _mulhilo(_PHILOX_M[0], c[0])
        hi1, lo1 = _mulhilo(_PHILOX_M[1], c[2])
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + _PHILOX_W[0]) & MASK32, (k1 + _PHILOX_W[1]) & MASK32
    return torch.stack(c, -1)


def philox(counter: torch.Tensor, key: int) -> torch.Tensor:
    """``philox4x32(seed=key, offset=counter)`` of common.cuh: 64-bit counter and key split into (low, high) words."""
    key &= MASK64
    return philox4x32_10(counter & MASK32, counter >> 32, 0, 0, key & MASK32, key >> 32)


def stream_bits(pos: torch.Tensor, key: int) -> torch.Tensor:
    """The 16 random bits of stream positions ``pos`` (int64): counter pos >> 3, word (pos & 7) >> 1, low half for even
    positions and high half for odd ones."""
    ctr = pos >> 3
    if pos.numel() == 0:
        return torch.zeros_like(pos)
    lo, hi = int(ctr.min()), int(ctr.max())
    if hi - lo < pos.numel():  # a dense range (every caller's case): one draw per counter instead of one per element
        words = philox(torch.arange(lo, hi + 1, dtype=torch.int64, device=pos.device), key).reshape(-1)
        w = words[(ctr - lo) * 4 + ((pos & 7) >> 1)]
    else:
        w = torch.gather(philox(ctr, key), -1, ((pos & 7) >> 1).unsqueeze(-1)).squeeze(-1)
    return (w >> (16 * (pos & 1))) & 0xFFFF


def sr_copy_bits(n: int, seed: int, device=None) -> torch.Tensor:
    """Random bits of ``sr_copy_`` for elements 0..n-1."""
    return stream_bits(torch.arange(n, dtype=torch.int64, device=device), seed)


def adamw_bits(pos: torch.Tensor, seed: int) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(p, exp_avg, exp_avg_sq) random bits at stream positions ``pos``: rng_base + element index for ``adamw_sr_multi_``,
    the global arena index for ``nvl_adamw_shard_``."""
    return (stream_bits(pos, seed), stream_bits(pos, seed + M_STATE), stream_bits(pos, seed + V_STATE))


def tensor_positions(n: int, rng_base: int, device=None) -> torch.Tensor:
    assert rng_base % 8 == 0, "the launch plan starts every tensor on a counter boundary"
    return rng_base + torch.arange(n, dtype=torch.int64, device=device)


# ----------------------------------------------------------------------------- bit patterns
def f32_bits(x: torch.Tensor) -> torch.Tensor:
    """fp32 bit pattern as a non-negative int64."""
    return x.float().contiguous().view(torch.int32).to(torch.int64) & MASK32


def bf16_bits(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().view(torch.int16).to(torch.int64) & 0xFFFF


def from_f32_bits(b: torch.Tensor) -> torch.Tensor:
    return (b - ((b >> 31) << 32)).to(torch.int32).view(torch.float32)


def from_bf16_bits(b: torch.Tensor) -> torch.Tensor:
    return (b - ((b >> 15) << 16)).to(torch.int16).view(torch.bfloat16)


def sr_bits(bits: torch.Tensor, r16: torch.Tensor) -> torch.Tensor:
    """bf16 bit pattern of the stochastic rounding of fp32 ``bits`` with random ``r16``.  Non-finite inputs keep their
    high half, a NaN with the bf16 quiet bit set when its payload would be dropped (a NaN of any payload is accepted by
    ``check_sr_exact``)."""
    nonfinite = (bits & 0x7F800000) == 0x7F800000
    special = (bits >> 16) | torch.where((bits & 0xFFFF) != 0, 0x40, 0)
    return torch.where(nonfinite, special, (bits + r16) >> 16)


def is_nan_bf16(b: torch.Tensor) -> torch.Tensor:
    return ((b & 0x7F80) == 0x7F80) & ((b & 0x7F) != 0)


# ----------------------------------------------------------------------------- fp64 AdamW
def bias_corrections(beta1: float, beta2: float, step: int) -> tuple[float, float]:
    """``adamw_sr_multi_``'s bias corrections: 1 - exp(step * log(beta)) in double, rounded to fp32 at the launch."""
    def bc(beta: float) -> float:
        return f32(1.0 - math.exp(step * math.log(beta))) if beta > 0 else 1.0
    return bc(beta1), bc(beta2)


def adamw_ref(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, *, lr: float, beta1: float,
              beta2: float, eps: float, wd: float, bc1: float, bc2: float, grad_scale: float | None = None):
    """fp64 AdamW of the exact inputs with the kernel's fp32 scalars (``bc1``/``bc2`` already fp32 values, see
    ``bias_corrections``).  Returns (p, p_bound, m, m_bound, v, v_bound): fp64 values of the kernel's fp32 results before
    rounding and absolute bounds on the kernel's error in them."""
    lr, b1, b2, eps, wd = (f32(x) for x in (lr, beta1, beta2, eps, wd))
    gs = 1.0 if grad_scale is None else f32(grad_scale)
    pd, gd, md, vd = (t.double() for t in (p, g, m, v))
    gd = gd * gs
    c = 1.0 - lr * wd
    pw0 = pd * c
    d_pw0 = pd.abs() * U32 * (lr * wd + abs(c)) + U32 * pw0.abs() + FTZ

    a, b = b1 * md, (1.0 - b1) * gd
    mn = a + b
    d_mn = 4 * U32 * (a.abs() + b.abs()) + 3 * FTZ
    a2, b2g = b2 * vd, (1.0 - b2) * gd * gd
    vn = a2 + b2g
    d_vn = 6 * U32 * (a2.abs() + b2g.abs()) + 3 * FTZ

    mh = mn / bc1
    d_mh = (d_mn + E_DIV * mn.abs()) / bc1 + FTZ
    vh = (vn / bc2).clamp_min(0.0)
    d_vh = (d_vn + E_DIV * vn.abs()) / bc2 + FTZ
    sq = vh.sqrt()
    d_sq0 = torch.minimum(d_vh.sqrt(), d_vh / sq.clamp_min(1e-300))
    d_sq = d_sq0 + E_SQRT * (sq + d_sq0)
    den = sq + eps
    d_den = d_sq + U32 * (den + d_sq)
    den_lo = torch.clamp_min(den - d_den, eps * (1 - U32))
    num = lr * mh
    d_num = lr * d_mh + U32 * (num.abs() + lr * d_mh) + FTZ
    upd = num / den
    d_q = (d_num * den + num.abs() * d_den) / (den * den_lo)
    d_upd = d_q + E_DIV * (upd.abs() + d_q) + FTZ
    pw = pw0 - upd
    d_p = d_pw0 + d_upd + U32 * (pw0.abs() + upd.abs() + d_pw0 + d_upd) + FTZ
    return pw, SECOND_ORDER * d_p, mn, SECOND_ORDER * d_mn, vn, SECOND_ORDER * d_vn


def adam_inputs(n: int, grad_dtype, state_dtype, gen: torch.Generator, device=None):
    """p ~ N(0, 1); per-element scale s = 10^U(-6, 0): g ~ N(0, s^2), m ~ N(0, (s / 3)^2), v ~ (N(0, s^2))^2, so that
    every regime from eps-dominated to large updates appears."""
    s = 10.0 ** (torch.rand(n, generator=gen, dtype=torch.float64, device=device) * 6 - 6)
    p = torch.randn(n, generator=gen, dtype=torch.float64, device=device).bfloat16()
    g = (torch.randn(n, generator=gen, dtype=torch.float64, device=device) * s).to(grad_dtype)
    m = (torch.randn(n, generator=gen, dtype=torch.float64, device=device) * s / 3).to(state_dtype)
    v = (torch.randn(n, generator=gen, dtype=torch.float64, device=device) * s).square().to(state_dtype)
    return p, g, m, v


# ----------------------------------------------------------------------------- checkers
def _ceil32(x: torch.Tensor) -> torch.Tensor:
    """Smallest fp32 >= x (x finite, within the fp32 range)."""
    f = x.float()
    return torch.where(f.double() >= x, f, torch.nextafter(f, torch.full_like(f, math.inf)))


def _floor32(x: torch.Tensor) -> torch.Tensor:
    f = x.float()
    return torch.where(f.double() <= x, f, torch.nextafter(f, torch.full_like(f, -math.inf)))


def _side(lo: torch.Tensor, hi: torch.Tensor, r16: torch.Tensor):
    """Range of bf16 magnitudes (15 bits) that SR with ``r16`` gives to the fp32 values in [lo, hi] (0 <= lo, or empty
    when hi < 0).  Returns (first, last, nonempty)."""
    big = torch.finfo(torch.float32).max
    lo_c, hi_c = lo.clamp(0.0, big), hi.clamp(max=big)
    first = (f32_bits(_ceil32(lo_c)) + r16) >> 16
    last = (f32_bits(_floor32(hi_c.clamp_min(0.0))) + r16) >> 16
    nonempty = (hi >= 0) & (_ceil32(lo_c) <= _floor32(hi_c.clamp_min(0.0)))
    return first, last, nonempty


def check_sr(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, r16: torch.Tensor, what: str = "") -> int:
    """Check a kernel's stochastically rounded bf16 ``out`` against every fp32 value within ``bound`` of ``ref``,
    rounded with the element's random bits ``r16``.  Where one bf16 value is possible the check is exact; the rest are
    *ambiguous*, and more than 2^-8 of them fails the check, so that it cannot pass vacuously (from 256 elements on:
    2^-8 of fewer is less than one element).  Returns the number of ambiguous elements."""
    out, ref, bound, r16 = out.reshape(-1), ref.reshape(-1), bound.reshape(-1), r16.reshape(-1)
    k = bf16_bits(out)
    sign, mag = k >> 15, k & 0x7FFF
    pf, pl, pn = _side(ref - bound, ref + bound, r16)
    nf, nl, nn = _side(-(ref + bound), -(ref - bound), r16)
    ok = ((sign == 0) & pn & (mag >= pf) & (mag <= pl)) | ((sign == 1) & nn & (mag >= nf) & (mag <= nl))
    if not bool(ok.all()):
        idx = (~ok).nonzero()[:5].flatten().tolist()
        vals = [(i, float(out[i]), float(ref[i]), float(bound[i])) for i in idx]
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements are not a stochastic rounding of the "
                             f"reference with their random bits; first (index, got, ref, bound): {vals}")
    choices = torch.where(pn, pl - pf + 1, 0) + torch.where(nn, nl - nf + 1, 0)
    amb = int((choices > 1).sum())
    if ok.numel() >= 256 and amb > MAX_AMBIGUOUS * ok.numel():
        raise AssertionError(f"{what}: {amb} of {ok.numel()} elements are ambiguous (more than {MAX_AMBIGUOUS:.3g}): "
                             "the bound is too loose for the check to mean anything")
    return amb


def check_sr_exact(out: torch.Tensor, src: torch.Tensor, r16: torch.Tensor, what: str = "") -> None:
    """``out`` (bf16) must equal the SR model of fp32 ``src`` bit for bit; where ``src`` is a NaN, ``out`` must be a NaN of
    the same sign."""
    bits = f32_bits(src.reshape(-1))
    want = sr_bits(bits, r16.reshape(-1))
    got = bf16_bits(out.reshape(-1))
    src_nan = torch.isnan(src.reshape(-1))
    ok = torch.where(src_nan, is_nan_bf16(got) & ((got >> 15) == (bits >> 31)), got == want)
    if not bool(ok.all()):
        idx = (~ok).nonzero()[:5].flatten().tolist()
        vals = [(i, hex(int(bits[i])), hex(int(want[i])), hex(int(got[i]))) for i in idx]
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements differ from the SR model; first "
                             f"(index, fp32 bits, expected, got): {vals}")


def check_adamw(p_out: torch.Tensor, m_out: torch.Tensor, v_out: torch.Tensor, p: torch.Tensor, g: torch.Tensor,
                m: torch.Tensor, v: torch.Tensor, pos: torch.Tensor, seed: int, what: str = "", **hyper) -> dict[str, float]:
    """Check one tensor's AdamW outputs: p (and bf16 states) with ``check_sr`` on their streams at positions ``pos``,
    fp32 states with ``assert_within``.  ``hyper``: the keyword arguments of ``adamw_ref``.  Returns
    ``{"p.ambiguous": ..., "m.ambiguous" or "m.err/bound": ..., ...}``."""
    pr, pb, mr, mb, vr, vb = adamw_ref(p, g, m, v, **hyper)
    rp, rm, rv = adamw_bits(pos, seed)
    stats = {"p.ambiguous": check_sr(p_out, pr, pb, rp, f"{what} p")}
    for name, out, ref, bound, r in (("m", m_out, mr, mb, rm), ("v", v_out, vr, vb, rv)):
        if out.dtype == torch.bfloat16:
            stats[f"{name}.ambiguous"] = check_sr(out, ref, bound, r, f"{what} {name}")
        else:
            stats[f"{name}.err/bound"] = assert_within(out, ref, bound, f"{what} {name}")
    return stats


def move_probability(ref: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """Probability that SR of the fp32 value nearest ``ref`` gives a bf16 other than ``p`` (|ref - p| under one bf16 ulp):
    the distance between the two bit patterns over 2^16."""
    d = (f32_bits(ref) - (bf16_bits(p) << 16)).abs()
    return (d.double() / 65536.0).clamp(max=1.0)
