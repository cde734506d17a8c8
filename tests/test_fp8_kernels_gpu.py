"""Every fp8 kernel against the fp64 models of ``tests/fp8_reference.py``, per element.

GEMMs: exact operands (codes from {-1, 0, +1}, fewer than 2^13 non-zero products per output element), so the only error
left is the fp32 scaling and the output rounding, at any K: every instance of ``gemm_fp8_kernel`` (ROWCOL with each
scale combination and scalar, MX with hand-built scale factors, BLOCKWISE bf16 / fp32, GROUPED_M store / accumulate,
GROUPED_K with its four epilogues) at M / N / K tails, K = 7168, a 16 384-deep reduction and more tiles than SMs, with
NaN past K in every operand row, canaried outputs and bitwise-reproducible runs.  Random operands at K <= 1024 with the
chain-length model, and the row-wise recipe's long weight-gradient reduction.

Quantisers: every code within the admissible range of the kernel's own scale, every scale within two ulp of
``max(amax / 448, 2^-126)``, at one-row / one-column / tail shapes, on strided inputs with NaN padding, and across the
whole fp32 range (groups at 2^-126 x {1, 7, 100, 447}, subnormal-only, all-zero and near the bf16 maximum).

Refused operands raise before anything is launched.
"""

import math

import pytest
import torch

from d9d_b200.kernel import fp8
from tests.fp8_reference import (
    FLT_MIN, U_BF16, U_CHAIN, U_F32, assert_codes_admissible, check_scales, code_rank, flush, gemm_bound, pack_mx_scales,
)
from tests.gemm_reference import Canaried, assert_within
from tests.test_fp8_experts_gpu import _layout_from_counts

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAN_CODE = 0x7F


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------ operands
def _pm1(rows, K, gen, *, sparse=False):
    """fp64 values from {-1, 0, +1}; ``sparse``: column 0 and every odd column zero (at most K/2 - 1 non-zero products
    per output element, so a 16 384-deep reduction stays below 2^13)."""
    v = torch.randint(-1, 2, (rows, K), generator=gen, device=DEV).double()
    if sparse:
        v[:, 1::2] = 0
        v[:, 0] = 0
    return v


def _fp8(v, *, pad=True):
    """e4m3 operand holding the exactly representable values ``v`` [rows, K]; ``pad``: row pitch rounded up past K to a
    multiple of 16 bytes plus 16, the padding filled with NaN codes (any read past K poisons the result)."""
    rows, K = v.shape
    codes = v.to(torch.float32).to(fp8.FP8).view(torch.uint8)
    if not pad:
        return codes.view(fp8.FP8)
    pitch = (K + 15) // 16 * 16 + 16
    buf = torch.full((rows, pitch), NAN_CODE, dtype=torch.uint8, device=DEV)
    buf[:, :K] = codes
    return buf.view(fp8.FP8)[:, :K]


def _scales(n, gen, lo_exp=-3, hi_exp=3):
    """Random fp32 scales (1 + u) * 2^e: almost never a power of two."""
    u = torch.rand(n, generator=gen, device=DEV)
    e = torch.randint(lo_exp, hi_exp + 1, (n,), generator=gen, device=DEV).float()
    return ((1 + u) * torch.exp2(e)).float()


def _blockwise_scales(groups, rows, gen, **kw):
    """k-block-major fp32 scales [groups, rows] with a row pitch of round_up(rows, 128), as the BLOCKWISE GEMM reads them."""
    s = torch.zeros(groups, (rows + 127) // 128 * 128, device=DEV)
    s[:, :rows] = _scales(groups * rows, gen, **kw).view(groups, rows)
    return s[:, :rows]


def _report(what, ratio):
    print(f"{what}: worst err / bound = {ratio:.3f}")


def _twice(run, out):
    """Runs ``run(view)`` into a canaried output and into a second one; asserts no stray writes and identical bits."""
    run(out.view)
    out.assert_untouched()
    again = Canaried(*out.view.shape, out.view.dtype, tma=True, device=DEV)
    run(again.view)
    assert torch.equal(out.view, again.view), "not bitwise reproducible"


# ------------------------------------------------------------------------------------------ ROWCOL
SHAPES = [(1, 16, 16), (16, 136, 127), (127, 128, 129), (129, 1000, 1000), (1000, 264, 7168), (8192, 4096, 256)]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("scales,scalar", [("both", 1.0), ("both", 0.3), ("none", 1.0), ("none", 0.3), ("a", 1.0), ("b", 0.3)])
def test_rowcol_exact_operands(ops, M, N, K, scales, scalar):
    g = _gen(M + N + K)
    A, B = _pm1(M, K, g), _pm1(N, K, g)
    sa = _scales(M, g) if scales in ("both", "a") else None
    sb = _scales(N, g) if scales in ("both", "b") else None
    ref = A @ B.t()
    S = A.abs() @ B.abs().t()
    col = lambda s: s.double()[:, None]  # noqa: E731
    row = lambda s: s.double()[None, :]  # noqa: E731
    if sa is not None:
        ref, S = ref * col(sa), S * col(sa)
    if sb is not None:
        ref, S = ref * row(sb), S * row(sb)
    ref, S = ref * scalar, S * abs(scalar)
    aq, bq = _fp8(A), _fp8(B)
    out = Canaried(M, N, torch.bfloat16, tma=True, device=DEV)
    _twice(lambda d: ops.gemm_fp8(aq, bq, sa, sb, scalar, d), out)
    r = assert_within(out.view, ref, gemm_bound(ref, S, K, K, torch.bfloat16, exact_chains=True), f"rowcol {M}x{N}x{K}")
    _report(f"rowcol exact M={M} N={N} K={K} scales={scales} scalar={scalar}", r)


def test_rowcol_exact_16k_reduction(ops):
    g = _gen(7)
    M, N, K = 256, 392, 16384
    A, B = _pm1(M, K, g, sparse=True), _pm1(N, K, g)
    sa, sb = _scales(M, g), _scales(N, g)
    ref = (A @ B.t()) * sa.double()[:, None] * sb.double()[None, :]
    S = (A.abs() @ B.abs().t()) * sa.double()[:, None] * sb.double()[None, :]
    aq, bq = _fp8(A), _fp8(B)
    out = Canaried(M, N, torch.bfloat16, tma=True, device=DEV)
    _twice(lambda d: ops.gemm_fp8(aq, bq, sa, sb, 1.0, d), out)
    _report("rowcol exact K=16384", assert_within(out.view, ref, gemm_bound(ref, S, K, K, torch.bfloat16, exact_chains=True), "K=16384"))


@pytest.mark.parametrize("M,N,K", [(256, 256, 256), (1000, 776, 528), (333, 128, 1024), (1, 16, 16)])
def test_rowcol_random_operands_chain_bound(ops, M, N, K):
    g = _gen(M * K)
    a = (torch.randn(M, K, generator=g, device=DEV) * torch.logspace(-2, 2, M, device=DEV)[:, None]).bfloat16()
    b = torch.randn(N, K, generator=g, device=DEV).bfloat16()
    aq, sa = ops.quantize_rowwise(a)
    bq, sb = ops.quantize_rowwise(b)
    A = aq.double() * sa.double()[:, None]
    B = bq.double() * sb.double()[:, None]
    ref, S = A @ B.t(), A.abs() @ B.abs().t()
    out = Canaried(M, N, torch.bfloat16, tma=True, device=DEV)
    _twice(lambda d: ops.gemm_fp8(aq, bq, sa, sb, 1.0, d), out)
    _report(f"rowcol random M={M} N={N} K={K}", assert_within(out.view, ref, gemm_bound(ref, S, K, K, torch.bfloat16), "rowcol random"))


def test_rowwise_weight_gradient_long_reduction(ops):
    """The row-wise recipe's weight gradient reduces over every token in one unpromoted chain.  Random inputs and
    round-to-nearest at U_CHAIN inside a chain give a norm-wise error of about U_CHAIN * sqrt((K + 1) / 6) for one chain
    and U_CHAIN * sqrt(129 / 6) for promoted 128-deep chains; the output is bf16, which alone costs about 2^-9 / sqrt(3)."""
    T, out_f, in_f = 16384, 576, 1536
    g = _gen(11)
    x = torch.randn(T, in_f, generator=g, device=DEV).bfloat16()
    dy = torch.randn(T, out_f, generator=g, device=DEV).bfloat16()
    dyq, sdy = ops.quantize_colwise_t(dy)
    xq, sx = ops.quantize_colwise_t(x)
    dw = torch.empty(out_f, in_f, device=DEV, dtype=torch.bfloat16)
    ops.gemm_fp8(dyq, xq, sdy, sx, 1.0, dw)
    exact = (dyq.double() * sdy.double()[:, None]) @ (xq.double() * sx.double()[:, None]).t()
    rel = float((dw.double() - exact).norm() / exact.norm())
    floor = float((exact.to(torch.bfloat16).double() - exact).norm() / exact.norm())
    one_chain, promoted = U_CHAIN * math.sqrt((T + 1) / 6), U_CHAIN * math.sqrt(129 / 6)
    print(f"rowwise wgrad {T} tokens: rel err {rel:.2e} (bf16 output rounding alone {floor:.2e}); "
          f"model: one chain {one_chain:.2e}, promoted {promoted:.2e}")
    assert rel <= 3 * one_chain


# ------------------------------------------------------------------------------------------ MX
@pytest.mark.parametrize("M,N,K", [(1, 16, 128), (127, 136, 256), (129, 1000, 1024), (1000, 128, 7168), (8192, 4096, 256)])
def test_mx_exact_operands(ops, M, N, K):
    g = _gen(M + 3 * N + K)
    A, B = _pm1(M, K, g), _pm1(N, K, g)
    ea = torch.randint(-8, 9, (M, K // 32), generator=g, device=DEV)
    eb = torch.randint(-8, 9, (N, K // 32), generator=g, device=DEV)
    As = A * torch.exp2(ea.double()).repeat_interleave(32, 1)
    Bs = B * torch.exp2(eb.double()).repeat_interleave(32, 1)
    ref, S = As @ Bs.t(), As.abs() @ Bs.abs().t()
    aq, bq = _fp8(A), _fp8(B)
    sfa, sfb = pack_mx_scales(ea), pack_mx_scales(eb)  # ceil(rows / 128) blocks: what the kernel reads
    out = Canaried(M, N, torch.bfloat16, tma=True, device=DEV)
    _twice(lambda d: ops.gemm_mxfp8(aq, sfa, bq, sfb, d), out)
    _report(f"mx exact M={M} N={N} K={K}", assert_within(out.view, ref, gemm_bound(ref, S, K, 32, torch.bfloat16, exact_chains=True), "mx"))


@pytest.mark.parametrize("M,N,K", [(256, 256, 256), (1000, 776, 512), (333, 128, 1024)])
def test_mx_random_operands_chain_bound(ops, M, N, K):
    g = _gen(M * K + 1)
    a = (torch.randn(M, K, generator=g, device=DEV) * torch.logspace(-3, 3, K // 32, device=DEV).repeat_interleave(32)).bfloat16()
    b = torch.randn(N, K, generator=g, device=DEV).bfloat16()
    aq, sfa = ops.quantize_mx(a)
    bq, sfb = ops.quantize_mx(b)
    A = fp8.dequantize_mx(aq, fp8.unpack_mx_scales(sfa, M, K)).double()
    B = fp8.dequantize_mx(bq, fp8.unpack_mx_scales(sfb, N, K)).double()
    ref, S = A @ B.t(), A.abs() @ B.abs().t()
    out = Canaried(M, N, torch.bfloat16, tma=True, device=DEV)
    _twice(lambda d: ops.gemm_mxfp8(aq, sfa, bq, sfb, d), out)
    _report(f"mx random M={M} N={N} K={K}", assert_within(out.view, ref, gemm_bound(ref, S, K, 32, torch.bfloat16), "mx random"))


# ------------------------------------------------------------------------------------------ BLOCKWISE
def _blockwise_ref(A, sa, B, sb):
    K = A.shape[1]
    ea = sa.double().repeat_interleave(128, 0)[:K].t()  # [M, K]
    eb = sb.double().repeat_interleave(128, 0)[:K].t()
    As, Bs = A * ea, B * eb
    return As @ Bs.t(), As.abs() @ Bs.abs().t()


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_blockwise_exact_operands(ops, M, N, K, dtype):
    g = _gen(M + 5 * N + K)
    A, B = _pm1(M, K, g), _pm1(N, K, g)
    G = (K + 127) // 128
    sa, sb = _blockwise_scales(G, M, g), _blockwise_scales(G, N, g)
    ref, S = _blockwise_ref(A, sa, B, sb)
    aq, bq = _fp8(A), _fp8(B)
    out = Canaried(M, N, dtype, tma=True, device=DEV)
    _twice(lambda d: ops.gemm_fp8_blockwise(aq, sa, bq, sb, d), out)
    _report(f"blockwise exact M={M} N={N} K={K} {dtype}",
            assert_within(out.view, ref, gemm_bound(ref, S, K, 128, dtype, exact_chains=True), "blockwise"))


# ------------------------------------------------------------------------------------------ grouped
@pytest.mark.parametrize("counts,K,N", [([1, 127, 128, 129, 0, 300], 1008, 136), ([4000, 4100], 256, 4096)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_grouped_m_exact_operands(ops, counts, K, N, accumulate):
    g = _gen(len(counts) + K + N)
    lay = _layout_from_counts(counts)
    E, cap = len(counts), lay.capacity
    A, B = _pm1(cap, K, g), _pm1(E * N, K, g)
    sa, sb = _scales(cap, g), _scales(E * N, g)
    aq, bq = _fp8(A, pad=False), _fp8(B, pad=False).view(E, N, K)
    canary = -7168.0
    base = torch.full((cap, N), canary, device=DEV, dtype=torch.bfloat16)
    if accumulate:
        base.normal_(generator=g)
    d, d2 = base.clone(), base.clone()
    ops.gemm_fp8_grouped_m(aq, sa, bq, sb, d, lay.tile_group, accumulate)
    ops.gemm_fp8_grouped_m(aq, sa, bq, sb, d2, lay.tile_group, accumulate)
    assert torch.equal(d, d2), "not bitwise reproducible"
    used = lay.tile_group.repeat_interleave(128) >= 0
    assert torch.equal(d[~used], base[~used])  # -1 tiles are never written
    As = A * sa.double()[:, None]
    Bs = (B * sb.double()[:, None]).view(E, N, K)
    prod = torch.zeros(cap, N, dtype=torch.float64, device=DEV)
    S = torch.zeros_like(prod)
    for t, e in enumerate(lay.tile_group.tolist()):
        if e >= 0:
            prod[128 * t : 128 * t + 128] = As[128 * t : 128 * t + 128] @ Bs[e].t()
            S[128 * t : 128 * t + 128] = As[128 * t : 128 * t + 128].abs() @ Bs[e].abs().t()
    rows = used.nonzero().squeeze(1)
    prod, S = prod[rows], S[rows]
    bound = gemm_bound(prod, S, K, 128, torch.bfloat16, exact_chains=True)
    ref = prod
    if accumulate:
        ref = prod + base[rows].double()
        bound = bound + U_BF16 * ref.abs()  # the reduce-add's rounding of d + rn_bf16(acc)
    _report(f"grouped_m exact counts={counts} K={K} N={N} acc={accumulate}", assert_within(d[rows], ref, bound, "grouped_m"))


@pytest.mark.parametrize("counts,M,N,sparse", [([1, 127, 128, 129, 0, 300], 136, 264, False), ([16000, 0, 5], 128, 192, True)])
@pytest.mark.parametrize("dtype,accumulate", [(torch.float32, False), (torch.float32, True), (torch.bfloat16, False),
                                              (torch.bfloat16, True)])
def test_grouped_k_exact_operands(ops, counts, M, N, sparse, dtype, accumulate):
    g = _gen(len(counts) + M + N)
    lay = _layout_from_counts(counts)
    E, cap = len(counts), lay.capacity
    seg = lay.seg_offsets.tolist()
    valid = torch.zeros(cap, dtype=torch.bool, device=DEV)
    for e, n in enumerate(counts):
        valid[seg[e] : seg[e] + n] = True
    # the transposed operands [M, cap] / [N, cap]: zeros outside the experts' rows, as quantize_segments_t writes them
    A = _pm1(cap, M, g, sparse=False).t().contiguous() * valid
    B = _pm1(cap, N, g).t().contiguous() * valid
    if sparse:
        A[:, 1::2] = 0
        A[:, 0] = 0
    sa, sb = _scales(E * M, g), _scales(E * N, g)
    aq, bq = _fp8(A, pad=False), _fp8(B, pad=False)
    base = torch.randn(E, M, N, generator=g, device=DEV).to(dtype)
    d, d2 = base.clone(), base.clone()
    ops.gemm_fp8_grouped_k(aq, sa, bq, sb, d, lay.seg_offsets, accumulate)
    ops.gemm_fp8_grouped_k(aq, sa, bq, sb, d2, lay.seg_offsets, accumulate)
    assert torch.equal(d, d2), "not bitwise reproducible"
    u_out = U_BF16 if dtype == torch.bfloat16 else U_F32
    worst = 0.0
    for e in range(E):
        cols = slice(seg[e], seg[e + 1])
        As = A[:, cols] * sa.view(E, M)[e].double()[:, None]
        Bs = B[:, cols] * sb.view(E, N)[e].double()[:, None]
        prod, S = As @ Bs.t(), As.abs() @ Bs.abs().t()
        if counts[e] == 0:
            want = base[e] if accumulate else torch.zeros_like(base[e])
            assert torch.equal(d[e], want), f"expert {e} without rows"
            continue
        bound = gemm_bound(prod, S, seg[e + 1] - seg[e], 128, dtype, exact_chains=True)
        ref = prod
        if accumulate:
            ref = prod + base[e].double()
            bound = bound + u_out * ref.abs()
        worst = max(worst, assert_within(d[e], ref, bound, f"grouped_k expert {e}"))
    _report(f"grouped_k exact counts={counts} M={M} N={N} {dtype} acc={accumulate}", worst)


# ------------------------------------------------------------------------------------------ GEMM dynamic range
def _tiny_scales(n, gen, exp):
    return _scales(n, gen, exp, exp)


def test_gemms_keep_results_whose_scale_product_is_subnormal(ops):
    """sa in [2^-60, 2^-59), sb in [2^-70, 2^-69): sa * sb is below 2^-126 and flushes, while (acc * sa) * sb is normal.
    Codes +-256: every partial sum is a multiple of 2^16 below 2^29 (exact), so every result is zero or at least 2^-114."""
    g = _gen(99)
    M, N, K = 256, 264, 384
    A, B = _pm1(M, K, g) * 256, _pm1(N, K, g) * 256
    aq, bq = _fp8(A), _fp8(B)
    sa, sb = _tiny_scales(M, g, -60), _tiny_scales(N, g, -70)
    ref = (A @ B.t()) * sa.double()[:, None] * sb.double()[None, :]
    S = (A.abs() @ B.abs().t()) * sa.double()[:, None] * sb.double()[None, :]
    d = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm_fp8(aq, bq, sa, sb, 1.0, d)
    _report("rowcol tiny scales", assert_within(d, ref, gemm_bound(ref, S, K, K, torch.bfloat16, exact_chains=True, flush_results=True), "rowcol"))
    # BLOCKWISE
    G = (K + 127) // 128
    sab, sbb = _blockwise_scales(G, M, g, lo_exp=-60, hi_exp=-60), _blockwise_scales(G, N, g, lo_exp=-70, hi_exp=-70)
    ref, S = _blockwise_ref(A, sab, B, sbb)
    for dtype in (torch.bfloat16, torch.float32):
        d = torch.empty(M, N, device=DEV, dtype=dtype)
        ops.gemm_fp8_blockwise(aq, sab, bq, sbb, d)
        _report(f"blockwise tiny scales {dtype}",
                assert_within(d, ref, gemm_bound(ref, S, K, 128, dtype, exact_chains=True, flush_results=True), "blockwise"))
    # MX: 2^-120 x 2^-10
    ea = torch.full((M, K // 32), -120, device=DEV)
    eb = torch.full((N, K // 32), -10, device=DEV)
    As, Bs = A * 2.0**-120, B * 2.0**-10
    ref, S = As @ Bs.t(), As.abs() @ Bs.abs().t()
    d = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm_mxfp8(aq, pack_mx_scales(ea), bq, pack_mx_scales(eb), d)
    _report("mx tiny scales", assert_within(d, ref, gemm_bound(ref, S, K, 32, torch.bfloat16, exact_chains=True, flush_results=True), "mx"))
    # GROUPED_M and GROUPED_K
    lay = _layout_from_counts([256])
    cap = lay.capacity
    Ag = torch.zeros(cap, K, device=DEV, dtype=torch.float64)
    Ag[:M] = A
    sag = _tiny_scales(cap, g, -60)
    d = torch.zeros(cap, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm_fp8_grouped_m(_fp8(Ag, pad=False), sag, _fp8(B, pad=False).view(1, N, K), sb, d, lay.tile_group, False)
    ref = (Ag[:M] @ B.t()) * sag[:M].double()[:, None] * sb.double()[None, :]
    S = (Ag[:M].abs() @ B.abs().t()) * sag[:M].double()[:, None] * sb.double()[None, :]
    _report("grouped_m tiny scales",
            assert_within(d[:M], ref, gemm_bound(ref, S, K, 128, torch.bfloat16, exact_chains=True, flush_results=True), "grouped_m"))
    # GROUPED_K: the expert's 256 rows are the reduction
    At = torch.zeros(M, cap, device=DEV, dtype=torch.float64)
    Bt = torch.zeros(N, cap, device=DEV, dtype=torch.float64)
    At[:, :256], Bt[:, :256] = A[:, :256], B[:, :256]
    dk = torch.zeros(1, M, N, device=DEV)
    ops.gemm_fp8_grouped_k(_fp8(At, pad=False), sa, _fp8(Bt, pad=False), sb, dk, lay.seg_offsets, False)
    ref = (At @ Bt.t()) * sa.double()[:, None] * sb.double()[None, :]
    S = (At.abs() @ Bt.abs().t()) * sa.double()[:, None] * sb.double()[None, :]
    _report("grouped_k tiny scales",
            assert_within(dk[0], ref, gemm_bound(ref, S, 256, 128, torch.float32, exact_chains=True, flush_results=True), "grouped_k"))


# ------------------------------------------------------------------------------------------ quantisers
def _x(rows, cols, seed, *, pad=0, spread=(-2, 2), dim=0):
    """bf16 [rows, cols] with magnitudes spread over 10^spread along ``dim`` (0: per row, 1: per column); ``pad``: row pitch
    cols + pad with NaN in the padding (any read past ``cols`` poisons a scale)."""
    g = _gen(seed)
    mag = torch.logspace(*spread, rows if dim == 0 else cols, device=DEV)
    v = torch.randn(rows, cols, generator=g, device=DEV) * (mag[:, None] if dim == 0 else mag[None, :])
    buf = torch.full((rows, cols + pad), float("nan"), device=DEV, dtype=torch.bfloat16)
    buf[:, :cols] = v.bfloat16()
    return buf[:, :cols]


def _check_rowwise(x, q, s, what):
    """Row groups: x [R, C], q [R, C], s [R]."""
    xf = flush(x)
    check_scales(s, xf.abs().amax(1), what, raw_amax=x.double().abs().amax(1))
    assert_codes_admissible(x, q, s[:, None], what)


def _check_transposed(x, qt, s, what):
    """Column groups with a transposed copy: x [R, C], qt [C, R], s [C]."""
    _check_rowwise(x.t(), qt, s, what)


def _check_blocked(x, q, s, what, gr, gc, transpose):
    """Groups of gr x gc elements of x [R, C]; q is x's copy ([R, C], or [C, R] with ``transpose``); s is k-block-major:
    s[c // gc, r] (plain copy) or s[r // gr, c] (transposed copy), each group's scale repeated on its rows / columns."""
    R, C = x.shape
    xf = flush(x).abs()
    Rp, Cp = -(-R // gr) * gr, -(-C // gc) * gc
    pad = torch.zeros(Rp, Cp, dtype=torch.float64, device=x.device)
    raw = pad.clone()
    pad[:R, :C], raw[:R, :C] = xf, x.double().abs()
    amax = pad.view(Rp // gr, gr, Cp // gc, gc).amax(dim=(1, 3))  # [R / gr, C / gc]
    raw_amax = raw.view(Rp // gr, gr, Cp // gc, gc).amax(dim=(1, 3))
    # the scale of every element of x, as the GEMM would apply it, from the layout the quantiser stored
    if transpose:
        s_elem = s.repeat_interleave(gr, 0)[:R]  # [R, C]: s[r // gr, c]
    else:
        s_elem = s.t().repeat_interleave(gc, 1)[:, :C]  # [R, C]: s[c // gc, r]
    g_amax = amax.repeat_interleave(gr, 0).repeat_interleave(gc, 1)[:R, :C]
    g_raw = raw_amax.repeat_interleave(gr, 0).repeat_interleave(gc, 1)[:R, :C]
    check_scales(s_elem, g_amax, what, raw_amax=g_raw)
    assert_codes_admissible(x, q.t() if transpose else q, s_elem, what)


def _check_mx(x, q, sf, what):
    M, K = x.shape
    e = fp8.unpack_mx_scales(sf, M, K)
    amax = flush(x).abs().view(M, K // 32, 32).amax(-1)
    raw = x.double().abs().view(M, K // 32, 32).amax(-1)  # a subnormal-only group: the kernel's max may or may not flush
    ok = (e == fp8.mx_scale_exponent(amax.float())) | (e == fp8.mx_scale_exponent(raw.float()))
    assert bool(ok.all()), f"{what}: scale exponents off at {(~ok).nonzero()[:4].tolist()}"  # exact integer arithmetic
    assert_codes_admissible(x, q, torch.exp2(e.double()).repeat_interleave(32, 1), what)


@pytest.mark.parametrize("M,K,pad", [(1, 16, 0), (3, 16, 8), (1000, 528, 0), (129, 4096, 16), (4097, 1008, 24)])
def test_quantize_rowwise_codes_and_scales(ops, M, K, pad):
    x = _x(M, K, M + K, pad=pad)
    if M > 2:
        x[M // 2] = 0
    q, s = ops.quantize_rowwise(x)
    assert q.shape == (M, K) and s.shape == (M,)
    _check_rowwise(x, q, s, f"quantize_rowwise {M}x{K}")


@pytest.mark.parametrize("R,C,pad", [(1, 64, 0), (777, 1, 7), (16, 16, 0), (1000, 520, 8), (129, 96, 32), (4100, 136, 0)])
def test_quantize_colwise_t_codes_and_scales(ops, R, C, pad):
    x = _x(R, C, R + C, pad=pad, dim=1)
    if C > 2:
        x[:, C // 2] = 0
    qt, s = ops.quantize_colwise_t(x)
    pitch = (R + 15) // 16 * 16
    assert qt.shape == (C, R) and qt.stride() == (pitch, 1)
    _check_transposed(x, qt, s, f"quantize_colwise_t {R}x{C}")
    full = qt.as_strided((C, pitch), (pitch, 1))
    assert not full[:, R:].view(torch.uint8).any()  # pad columns are zero codes


@pytest.mark.parametrize("E,R,C", [(3, 16, 1), (2, 144, 200), (5, 64, 48)])
def test_quantize_colwise_t_batched_codes_and_scales(ops, E, R, C):
    x = torch.stack([_x(R, C, 10 * e + R, dim=1) for e in range(E)])
    x[0, :, 0] = 0
    q, s = ops.quantize_colwise_t_batched(x)
    assert q.shape == (E, C, R) and s.shape == (E, C)
    for e in range(E):
        _check_transposed(x[e], q[e], s[e], f"quantize_colwise_t_batched plane {e}")


def test_quantize_segments_t_codes_and_scales(ops):
    counts = [0, 1, 127, 128, 129, 0, 300, 5]
    lay = _layout_from_counts(counts)
    C = 80
    x = _x(lay.capacity, C, 5, dim=1)
    seg = lay.seg_offsets.tolist()
    for e, n in enumerate(counts):  # pad rows hold NaN: they must come out as zero codes and not reach a scale
        x[seg[e] + n : seg[e + 1]] = float("nan")
    x[seg[-1]:] = float("nan")
    x[seg[6] : seg[6] + 300, 7] = 0
    q, s = ops.quantize_segments_t(x, lay.tile_group, lay.seg_offsets, lay.counts)
    assert q.shape == (C, lay.capacity) and s.shape == (len(counts), C)
    valid = torch.zeros(lay.capacity, dtype=torch.bool, device=DEV)
    for e, n in enumerate(counts):
        valid[seg[e] : seg[e] + n] = True
        if n == 0:
            assert bool((s[e] == 1).all()), f"expert {e} without rows"
            continue
        rows = slice(seg[e], seg[e] + n)
        _check_transposed(x[rows], q[:, rows], s[e], f"quantize_segments_t expert {e}")
    assert not q[:, ~valid].view(torch.uint8).any()  # exact zeros outside the experts' rows


@pytest.mark.parametrize("M,K,pad", [(1, 16, 0), (3, 16, 8), (130, 400, 0), (1000, 576, 16)])
def test_quantize_blockwise_row_groups(ops, M, K, pad):
    x = _x(M, K, M + K, pad=pad, dim=1)
    if M > 2:
        x[M // 2] = 0
    q, s = ops.quantize_blockwise(x)
    _check_blocked(x, q, s, f"quantize_blockwise {M}x{K}", 1, 128, False)


@pytest.mark.parametrize("M,C,pad", [(1, 16, 0), (5, 32, 0), (130, 144, 8), (1000, 576, 0), (16384, 64, 0)])
def test_quantize_blockwise_t_token_groups(ops, M, C, pad):
    x = _x(M, C, M + C, pad=pad)
    if C > 4:
        x[:, 3] = 0
    qt, s = ops.quantize_blockwise_t(x)
    pitch = (M + 15) // 16 * 16
    assert qt.shape == (C, M) and qt.stride() == (pitch, 1)
    _check_blocked(x, qt, s, f"quantize_blockwise_t {M}x{C}", 128, 1, True)
    assert not qt.as_strided((C, pitch), (pitch, 1))[:, M:].view(torch.uint8).any()  # pad columns are zero codes


@pytest.mark.parametrize("N,K", [(16, 16), (144, 400), (576, 7168), (272, 144)])
def test_quantize_weight_blocks_both_copies(ops, N, K):
    w = _x(N, K, N + K, spread=(-2, 1))
    q, s = ops.quantize_weight_blocks(w)
    qt, st = ops.quantize_weight_blocks(w, True)
    _check_blocked(w, q, s, f"quantize_weight_blocks {N}x{K}", 128, 128, False)
    _check_blocked(w.t(), qt, st, f"quantize_weight_blocks^T {N}x{K}", 128, 128, False)
    assert torch.equal(qt.view(torch.uint8), q.view(torch.uint8).t())


@pytest.mark.parametrize("M,K,pad", [(1, 128, 0), (300, 1024, 16), (129, 256, 0)])
def test_quantize_mx_codes_and_scales(ops, M, K, pad):
    g = _gen(M + K)
    x = (torch.randn(M, K, generator=g, device=DEV) * torch.logspace(-3, 3, K // 32, device=DEV).repeat_interleave(32)).bfloat16()
    buf = torch.full((M, K + pad), float("nan"), device=DEV, dtype=torch.bfloat16)
    buf[:, :K] = x
    x = buf[:, :K]
    x[0, 32:64] = 0
    q, sf = ops.quantize_mx(x)
    _check_mx(x, q, sf, f"quantize_mx {M}x{K}")


# ------------------------------------------------------------------------------------------ quantiser dynamic range
LEVELS = [1.0, FLT_MIN, 7 * FLT_MIN, 100 * FLT_MIN, 447 * FLT_MIN, 2.0**-130, 0.0, 3.0e38]  # 2^-130: subnormal-only


def _range_rows(cols, seed):
    """bf16 [len(LEVELS), cols]: row i has amax LEVELS[i] (one element exactly at it, the rest uniform below it)."""
    g = _gen(seed)
    u = torch.rand(len(LEVELS), cols, generator=g, device=DEV, dtype=torch.float64) * 2 - 1
    u[:, 0] = 1.0
    x = (u * torch.tensor(LEVELS, device=DEV, dtype=torch.float64)[:, None]).bfloat16()
    assert bool(torch.isfinite(x).all())
    return x


def _assert_finite_codes(q):
    assert not bool((code_rank(q.view(torch.uint8)).abs() > 126).any()), "NaN codes"


def test_quantisers_across_the_fp32_range(ops):
    """Groups whose amax is 2^-126 x {1, 7, 100, 447}, subnormal-only, all-zero and near the bf16 maximum: every code is
    finite, every scale finite and positive, every element at or above 2^-126 within its admissible codes."""
    X = _range_rows(256, 1)  # row groups
    q, s = ops.quantize_rowwise(X)
    _assert_finite_codes(q)
    _check_rowwise(X, q, s, "quantize_rowwise range")
    q, s = ops.quantize_blockwise(X)
    _assert_finite_codes(q)
    _check_blocked(X, q, s, "quantize_blockwise range", 1, 128, False)
    q, sf = ops.quantize_mx(X)
    _assert_finite_codes(q)
    _check_mx(X, q, sf, "quantize_mx range")
    Xt = X.t().contiguous()  # column groups: [256, 8]
    qt, s = ops.quantize_colwise_t(Xt)
    _assert_finite_codes(qt)
    _check_transposed(Xt, qt, s, "quantize_colwise_t range")
    qb, sb = ops.quantize_colwise_t_batched(torch.stack([Xt, Xt.flip(1)]))
    _assert_finite_codes(qb)
    _check_transposed(Xt, qb[0], sb[0], "quantize_colwise_t_batched range")
    _check_transposed(Xt.flip(1), qb[1], sb[1], "quantize_colwise_t_batched range (plane 1)")
    lay = _layout_from_counts([256])
    xs = torch.zeros(lay.capacity, 8, device=DEV, dtype=torch.bfloat16)
    xs[:256] = Xt
    qs, ss = ops.quantize_segments_t(xs, lay.tile_group, lay.seg_offsets, lay.counts)
    _assert_finite_codes(qs)
    _check_transposed(Xt, qs[:, :256], ss[0], "quantize_segments_t range")
    Xc = Xt.repeat(1, 2)  # [256, 16]: blockwise_t needs 16 columns
    qt, s = ops.quantize_blockwise_t(Xc)
    _assert_finite_codes(qt)
    _check_blocked(Xc, qt, s, "quantize_blockwise_t range", 128, 1, True)
    # 128 x 128 weight blocks: block j of a [128, 8 * 128] weight has amax LEVELS[j]
    W = _range_rows(128 * 128, 2).view(len(LEVELS), 128, 128).permute(1, 0, 2).reshape(128, len(LEVELS) * 128).contiguous()
    q, s = ops.quantize_weight_blocks(W)
    qt, st = ops.quantize_weight_blocks(W, True)
    _assert_finite_codes(q)
    _assert_finite_codes(qt)
    _check_blocked(W, q, s, "quantize_weight_blocks range", 128, 128, False)
    _check_blocked(W.t(), qt, st, "quantize_weight_blocks^T range", 128, 128, False)


# ------------------------------------------------------------------------------------------ refused operands
def _refused(calls, *watch):
    before = [w.clone() for w in watch]
    for i, f in enumerate(calls):
        with pytest.raises((RuntimeError, ValueError)):
            f()
            print(f"call {i} was not refused")
    torch.cuda.synchronize()
    for w, b in zip(watch, before):
        assert torch.equal(w.view(torch.uint8), b.view(torch.uint8)), "a refused call wrote its output"


def test_gemm_fp8_and_gemm_mxfp8_refuse_bad_operands(ops):
    M, N, K = 200, 144, 256
    g = _gen(3)
    aq, bq = _fp8(_pm1(M, K, g), pad=False), _fp8(_pm1(N, K, g), pad=False)
    sa, sb = _scales(M, g), _scales(N, g)
    d = torch.full((M, N), -7168.0, device=DEV, dtype=torch.bfloat16)
    unaligned = _fp8(_pm1(M, 40, g), pad=False)  # K = 40: 40-byte rows, not a multiple of 16
    mis = torch.empty(M, N + 8, device=DEV, dtype=torch.bfloat16)[:, 1 : N + 1]
    _refused([
        lambda: ops.gemm_fp8(aq.view(torch.uint8), bq, sa, sb, 1.0, d),  # dtype
        lambda: ops.gemm_fp8(aq.float(), bq, sa, sb, 1.0, d),
        lambda: ops.gemm_fp8(aq, bq, sa[:-1], sb, 1.0, d),  # scale length
        lambda: ops.gemm_fp8(aq, bq, sa, sb[:-1], 1.0, d),
        lambda: ops.gemm_fp8(aq, bq, sa.double(), sb, 1.0, d),  # scale dtype
        lambda: ops.gemm_fp8(aq, bq, sa.cpu(), sb, 1.0, d),  # host-resident scales
        lambda: ops.gemm_fp8(aq, bq, sa, sb.cpu(), 1.0, d),
        lambda: ops.gemm_fp8(unaligned, _fp8(_pm1(N, 40, g), pad=False), sa, sb, 1.0, d),  # K rows not 16-byte aligned
        lambda: ops.gemm_fp8(aq, bq[:, :128], sa, sb, 1.0, d),  # K mismatch
        lambda: ops.gemm_fp8(aq, bq, sa, sb, 1.0, mis),  # misaligned output
        lambda: ops.gemm_fp8(aq, bq, sa, sb, 1.0, d[:-1]),  # mis-shaped output
        lambda: ops.gemm_fp8(aq, bq, sa, sb, 1.0, d.float()),  # fp32 output
    ], d)
    ea, eb = torch.zeros(M, K // 32, device=DEV, dtype=torch.int64), torch.zeros(N, K // 32, device=DEV, dtype=torch.int64)
    sfa, sfb = pack_mx_scales(ea), pack_mx_scales(eb)
    a64, b64 = _fp8(_pm1(M, 64, g), pad=False), _fp8(_pm1(N, 64, g), pad=False)
    _refused([
        lambda: ops.gemm_mxfp8(a64, sfa, b64, sfb, d),  # K not a multiple of 128
        lambda: ops.gemm_mxfp8(aq, sfa[:1], bq, sfb, d),  # too few scale blocks
        lambda: ops.gemm_mxfp8(aq, sfa, bq, sfb[:, :1], d),
        lambda: ops.gemm_mxfp8(aq, sfa.int(), bq, sfb, d),  # scale dtype
        lambda: ops.gemm_mxfp8(aq, sfa.cpu(), bq, sfb, d),  # host-resident scales
        lambda: ops.gemm_mxfp8(aq.float(), sfa, bq, sfb, d),  # operand dtype
        lambda: ops.gemm_mxfp8(aq, sfa, bq, sfb, mis),  # misaligned output
        lambda: ops.gemm_mxfp8(aq, sfa, bq, sfb, d[:, :-8]),  # mis-shaped output
    ], d)


def test_quantisers_refuse_bad_operands(ops):
    x = torch.randn(64, 256, device=DEV).bfloat16()
    off = torch.randn(64 * 256 + 1, device=DEV).bfloat16()[1:].view(64, 256)  # 2 bytes past a 16-byte boundary
    _refused([
        lambda: ops.quantize_rowwise(x.float()),  # dtype
        lambda: ops.quantize_rowwise(x[:, :40]),  # K not a multiple of 16
        lambda: ops.quantize_rowwise(off),  # misaligned rows
        lambda: ops.quantize_rowwise(x.cpu()),
        lambda: ops.quantize_rowwise(x.view(4, 16, 256)),
        lambda: ops.quantize_colwise_t(x.float()),
        lambda: ops.quantize_colwise_t(x.t()),  # column stride != 1
        lambda: ops.quantize_colwise_t(x.cpu()),
        lambda: ops.quantize_colwise_t(x.view(4, 16, 256)),
        lambda: ops.quantize_mx(x[:, :64]),  # K not a multiple of 128
        lambda: ops.quantize_mx(x.float()),
        lambda: ops.quantize_mx(off),
        lambda: ops.quantize_mx(x.cpu()),
    ])
