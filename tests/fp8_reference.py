"""fp64 models of the fp8 (e4m3) quantisers and GEMMs.  Pure torch: works on CPU tensors (self-test) and CUDA tensors.

Quantisers.  A kernel computes ``code = rn_e4m3(fl32(x * rcp(s)))``: the reciprocal has at most one ulp of error and the
product one fp32 rounding, so the code lies between ``rn_e4m3(x / s * (1 - delta))`` and ``rn_e4m3(x / s * (1 + delta))``
with ``delta = 2^-21`` (:func:`admissible_codes`).  ``rn_e4m3`` is modelled here from the 256-code table, independently
of torch's float8 cast.  The library builds with flush-to-zero, so an element below 2^-126 may come out as a zero code
and does not count towards its group's amax.  The scale of a group is ``max(amax / 448, 2^-126)`` to within two ulp
(``div.approx``), and exactly 1 for an all-zero group (:func:`check_scales`).

GEMMs.  For ``D = (A @ B^T) * scales`` with the fp64 product ``ref`` of the codes and scales the kernel consumed and
``S = |A| @ |B|^T`` (scaled), an accumulation in chains of length L at a unit roundoff ``U_CHAIN`` whose results are
added and scaled in fp32 errs by at most

    L * U_CHAIN * S + (ceil(K / L) + 3) * U_F32 * S + output rounding

(:func:`gemm_bound`).  L is K for the row / column-scaled dense GEMM (one chain), 32 for MX and 128 for the blockwise
and grouped GEMMs.  With operand codes from {-1, 0, +1} and fewer than 2^13 non-zero products per output element, every
partial sum is an integer below 2^13 and exact in any order under any accumulator of 14 or more bits: the chain term
drops out (``exact_chains=True``) and the bound holds at any K.
"""

from __future__ import annotations

import math

import torch

from tests.gemm_reference import U_BF16, U_F32

U_CHAIN = 2.0**-13  # modelled unit roundoff of the tensor core's e4m3 accumulation inside one MMA chain
FLT_MIN = 2.0**-126
E4M3_MAX = 448.0
DELTA = 2.0**-21  # relative error of fl32(x * rcp.approx(s)) against x / s
FLUSH_RESULT = 2.0**-118  # GEMM results below this may flush to zero (one of the fp32 scale products is subnormal)
NAN_RANK = 1 << 20  # rank given to the NaN codes 0x7f / 0xff: outside every admissible range


def e4m3_values() -> torch.Tensor:
    """fp64 value of each of the 256 codes (NaN for 0x7f and 0xff): sign bit 7, exponent bits 6..3 (bias 7), mantissa
    bits 2..0; exponent 0 is subnormal (m / 8 * 2^-6)."""
    out = []
    for c in range(256):
        sign = -1.0 if c & 0x80 else 1.0
        e, m = (c >> 3) & 0xF, c & 7
        if e == 15 and m == 7:
            out.append(math.nan)
        elif e == 0:
            out.append(sign * m / 8 * 2.0**-6)
        else:
            out.append(sign * (1 + m / 8) * 2.0 ** (e - 7))
    return torch.tensor(out, dtype=torch.float64)


_MAGS = e4m3_values()[:127]  # codes 0x00 .. 0x7e: the non-negative finite values, increasing (0 .. 448)


def rn_e4m3(v: torch.Tensor) -> torch.Tensor:
    """Codes (int64, 0 .. 255) of ``v`` rounded to nearest e4m3, ties to even, saturating at +-448 (what
    ``cvt.rn.satfinite.e4m3x2.f32`` does).  ``v`` must be finite; -0 and negative values that round to 0 give 0x80."""
    v = v.double()
    mags = _MAGS.to(v.device)
    a = v.abs().clamp_max(E4M3_MAX).contiguous()
    hi = torch.searchsorted(mags, a).clamp_max(126)  # first magnitude >= a
    lo = (hi - 1).clamp_min(0)
    dlo, dhi = a - mags[lo], mags[hi] - a
    pick_hi = (dhi < dlo) | ((dhi == dlo) & (hi % 2 == 0))
    code = torch.where(pick_hi, hi, lo)
    return torch.where(torch.signbit(v), code | 0x80, code)


def code_rank(codes: torch.Tensor) -> torch.Tensor:
    """Codes -> signed ordinal (int64): e4m3 codes of one sign are ordered like their magnitudes, so ``-(c & 0x7f)`` for
    negative codes and ``c`` otherwise orders every finite code by value, with +0 and -0 both at 0.  NaN codes map to
    +-NAN_RANK."""
    c = codes.to(torch.int64) & 0xFF
    mag = c & 0x7F
    mag = torch.where(mag == 0x7F, torch.full_like(mag, NAN_RANK), mag)
    return torch.where(c & 0x80 != 0, -mag, mag)


def flush(x: torch.Tensor) -> torch.Tensor:
    """fp64 copy of ``x`` with magnitudes below 2^-126 set to zero (flush-to-zero)."""
    x = x.double()
    return torch.where(x.abs() < FLT_MIN, torch.zeros_like(x), x)


def admissible_codes(x: torch.Tensor, s: torch.Tensor, delta: float = DELTA) -> tuple[torch.Tensor, torch.Tensor]:
    """(lowest, highest) code rank that ``rn_e4m3(x / s * (1 +- delta))`` can give; ``x`` and ``s`` broadcast.  An element
    below 2^-126 may also give a zero code (flush-to-zero)."""
    v = x.double() / s.double()
    r1, r2 = code_rank(rn_e4m3(v * (1 - delta))), code_rank(rn_e4m3(v * (1 + delta)))
    lo, hi = torch.minimum(r1, r2), torch.maximum(r1, r2)
    tiny = x.double().abs() < FLT_MIN
    return torch.where(tiny, lo.clamp_max(0), lo), torch.where(tiny, hi.clamp_min(0), hi)


def assert_codes_admissible(x: torch.Tensor, q: torch.Tensor, s: torch.Tensor, what: str = "", delta: float = DELTA) -> None:
    """Every code of ``q`` (float8_e4m3fn or uint8, same shape as ``x``) within :func:`admissible_codes` of ``x`` and the
    scale ``s`` the kernel reported (broadcast to ``x``)."""
    lo, hi = admissible_codes(x, s, delta)
    r = code_rank(q.view(torch.uint8) if q.dtype != torch.uint8 else q)
    bad = (r < lo) | (r > hi)
    if bool(bad.any()):
        idx = bad.nonzero()[:5].tolist()
        xb = x.double().expand_as(bad)
        sb = s.double().expand_as(bad)
        vals = [(i, float(xb[tuple(i)]), float(sb[tuple(i)]), int(r[tuple(i)]), int(lo[tuple(i)]), int(hi[tuple(i)])) for i in idx]
        raise AssertionError(f"{what}: {int(bad.sum())} codes outside the admissible range, first (index, x, s, rank, lo, hi): {vals}")


def _ulp32(v: torch.Tensor) -> torch.Tensor:
    """fp32 ulp at |v| (normal range; 2^-149 below it)."""
    _, e = torch.frexp(v.double().abs().clamp_min(FLT_MIN))
    return torch.exp2((e - 24).double())


def scale_bounds(amax: torch.Tensor, *, ulps: int = 2) -> tuple[torch.Tensor, torch.Tensor]:
    """Admissible [lo, hi] of the scale of a group with the given amax (fp64, already flushed): ``max(amax / 448, 2^-126)``
    within ``ulps`` fp32 ulp, exactly 1 for an all-zero group."""
    t = (amax.double() / E4M3_MAX).clamp_min(FLT_MIN)
    u = ulps * _ulp32(t)
    zero = amax == 0
    lo = torch.where(zero, torch.ones_like(t), (t - u).clamp_min(FLT_MIN))
    hi = torch.where(zero, torch.ones_like(t), t + u)
    return lo, hi


def check_scales(s: torch.Tensor, amax: torch.Tensor, what: str = "", *, raw_amax: torch.Tensor | None = None) -> None:
    """Kernel scales ``s`` against the flushed group amax.  A group whose elements are all below 2^-126 but not all zero
    (``raw_amax > 0``) may also get the floor 2^-126 instead of 1, depending on whether the kernel's max flushes."""
    s = s.double()
    assert bool(torch.isfinite(s).all()) and bool((s > 0).all()), f"{what}: non-finite or non-positive scale"
    lo, hi = scale_bounds(amax)
    ok = (s >= lo) & (s <= hi)
    if raw_amax is not None:
        ok |= (amax == 0) & (raw_amax.double() > 0) & (s == FLT_MIN)
    if not bool(ok.all()):
        idx = (~ok).nonzero()[:5].tolist()
        vals = [(i, float(s[tuple(i)]), float(amax[tuple(i)]), float(lo[tuple(i)]), float(hi[tuple(i)])) for i in idx]
        raise AssertionError(f"{what}: {int((~ok).sum())} scales off, first (index, s, amax, lo, hi): {vals}")


# ----------------------------------------------------------------------------- MX scale factors
def pack_mx_scales(e: torch.Tensor, row_blocks: int | None = None) -> torch.Tensor:
    """Exponents ``[rows, K/32]`` (int, -127 .. 127) -> the UE8M0 block layout ``[row_blocks, K/128, 512]`` (byte
    ``(r%32)*16 + (r//32)*4 + g``) that the MXFP8 GEMM reads; the inverse of ``fp8.unpack_mx_scales``.  Rows past
    ``rows`` get exponent 0."""
    rows, groups = e.shape
    nb = row_blocks if row_blocks is not None else (rows + 127) // 128
    kb = groups // 4
    full = torch.zeros(nb * 128, groups, dtype=torch.int64, device=e.device)
    full[:rows] = e.to(torch.int64)
    b = (full + 127).to(torch.uint8).view(nb, 4, 32, kb, 4)  # [blk, r//32, r%32, kblock, g]
    return b.permute(0, 3, 2, 1, 4).contiguous().view(nb, kb, 512)


# ----------------------------------------------------------------------------- GEMM
def gemm_bound(ref: torch.Tensor, S: torch.Tensor, K: int, chain: int, out_dtype: torch.dtype, *,
               exact_chains: bool = False, flush_results: bool = False) -> torch.Tensor:
    """Per-element bound on |D - ref| (see the module docstring).  ``flush_results``: results below 2^-118 may also
    come out as zero."""
    f = (math.ceil(K / chain) + 3) * U_F32 * S
    if not exact_chains:
        f = f + chain * U_CHAIN * S
    u_out = U_BF16 if out_dtype == torch.bfloat16 else U_F32
    bound = f + u_out * (ref.abs() + f)
    if flush_results:
        bound = torch.where(ref.abs() < FLUSH_RESULT, torch.maximum(bound, ref.abs()), bound)
    return bound
