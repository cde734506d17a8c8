"""Per-element fp64 checks of the bandwidth-bound kernels: RMSNorm, SiLU·mul(·probs), RoPE, fused q/k RMSNorm + RoPE,
MoE layout / permute / gather and the gradient utilities (``ops/csrc/elementwise.cu``, ``qk_norm_rope.cu``, ``moe.cu``).

Every kernel here is grid-stride or persistent with a capped grid.  The "persistent" sizes are computed from the SM
count with the same caps as the launchers (cited next to each), so that every block runs at least three passes plus a
ragged tail.  The exact probes feed integer-valued data (and inv_rms = 1, quarter-turn angles) so that every product and
partial sum is exact in fp32: the result must then match the fp64 reference bit for bit, which catches a lost or
duplicated row / warp / block partial that a worst-case bound over 10^5 rows cannot see."""

from __future__ import annotations

import math

import pytest
import torch

from tests.gemm_reference import assert_within
from tests.pointwise_reference import (
    U32,
    moe_gather_ref,
    qk_norm_rope_bwd_ref,
    qk_norm_rope_fwd_ref,
    rms_norm_bwd_ref,
    rms_norm_fwd_ref,
    rope_ref,
    rounding,
    silu_mul_bwd_ref,
    silu_mul_fwd_ref,
    silu_mul_probs_bwd_ref,
    silu_mul_probs_fwd_ref,
    sumsq_ref,
)

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float32, torch.float16]
EPS = 1e-6
WORST: dict[str, float] = {}


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    yield _ops.load()
    if WORST:
        print("\nworst err/bound per op: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def check(op: str, d: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> None:
    r = assert_within(d, ref, bound, op)
    WORST[op] = max(WORST.get(op, 0.0), r)


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ints(shape, lo, hi, dtype, gen=None):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=gen).to(dtype)


def _signs(shape, dtype):
    return (torch.randint(0, 2, shape, device="cuda") * 2 - 1).to(dtype)


# ============================================================================ RMSNorm
def _rms_geometry(N: int, fwd: bool) -> tuple[int, int]:
    """(rows per block per pass, rows per grid pass) of the launch elementwise.cu picks for N."""
    if fwd:
        if N <= 2048:
            # D9D_RMS_FWD_DISPATCH (elementwise.cu:541-546): G lanes per row, VPL vectors per lane, U = 2 row groups per
            # warp when VPL <= 2 (rms_fwd_kernel, elementwise.cu:121-122); 8 warps per block, at most num_sms * 8 blocks
            # (rms_fwd_launch, elementwise.cu:290)
            G = 8 if N <= 64 else 16 if N <= 128 else 32
            vpl = 1 if N <= 256 else 2 if N <= 512 else 4 if N <= 1024 else 8
            per_block = 8 * (32 // G) * (2 if vpl <= 2 else 1)
            return per_block, per_block * sms() * 8
        return 1, sms() * 16  # rms_fwd_block_launch: one row per block, num_sms * 16 blocks (elementwise.cu:506)
    # backward: at most rms_norm_bwd_num_partials() = num_sms * 8 resident blocks (elementwise.cu:306, 519, 531, 568)
    if N <= 1024:  # rms_bwd_launch: 8 warps of 32 / G rows
        G = 8 if N <= 64 else 16 if N <= 128 else 32
        return 8 * (32 // G), 8 * (32 // G) * sms() * 8
    return 1, sms() * 8  # rms_bwd_block_launch: one row per block


def _rms_persistent_rows(N: int) -> int:
    passes = [_rms_geometry(N, True)[1]] + ([_rms_geometry(N, False)[1]] if N <= 8192 else [])
    return 3 * max(passes) + 5


RMS_N = [8, 64, 72, 128, 136, 256, 264, 512, 520, 1024, 1032, 2048, 2056, 4096, 4104, 8192, 8200, 16384]


@pytest.mark.parametrize("N", RMS_N)
@pytest.mark.parametrize("M", [1, 7, 517, "persistent"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("zc", [False, True])
def test_rms_norm(ops, N, M, dtype, zc):
    """Every forward bucket (9) and backward bucket (8) at its upper edge and at a width that leaves lanes idle; the
    backward takes the forward's inv_rms, so each pass is checked by itself.  N > 8192 has no backward."""
    if M == "persistent":
        if zc:
            pytest.skip("the persistent sizes run once per (N, dtype)")
        M = _rms_persistent_rows(N)
    gen = torch.Generator(device="cuda").manual_seed(N * 31 + M)
    x = (torch.randn(M, N, device="cuda", generator=gen) * (torch.rand(M, 1, device="cuda", generator=gen) * 4 + 0.05)).to(dtype)
    w = (torch.randn(N, device="cuda", generator=gen) * 0.1 + (0.0 if zc else 1.0)).to(dtype)
    out, inv = ops.rms_norm_fwd(x, w, EPS, zc)
    ref, bound, ir_ref, ir_bound = rms_norm_fwd_ref(x, w, EPS, zc, inv_rms=inv)
    check("rms_norm_fwd.inv_rms", inv, ir_ref, ir_bound)
    check("rms_norm_fwd.out", out, ref, bound)
    del ref, bound
    if N > 8192:
        with pytest.raises(RuntimeError, match="N > 8192"):
            ops.rms_norm_bwd(out, x, w, inv, zc)
        return
    dy = torch.randn(M, N, device="cuda", generator=gen).to(dtype)
    dx, dw = ops.rms_norm_bwd(dy, x, w, inv, zc)
    dx_ref, dx_b, dw_ref, dw_b = rms_norm_bwd_ref(dy, x, w, inv, zc)
    check("rms_norm_bwd.dx", dx, dx_ref, dx_b)
    check("rms_norm_bwd.dw", dw, dw_ref, dw_b)
    if M > 517:
        _, dw2 = ops.rms_norm_bwd(dy, x, w, inv, zc)
        assert torch.equal(dw.view(torch.int16 if dw.element_size() == 2 else torch.int32),
                           dw2.view(torch.int16 if dw.element_size() == 2 else torch.int32)), "dw reduction is not deterministic"


@pytest.mark.parametrize("dtype", DTYPES)
def test_rms_norm_autograd_end_to_end(ops, dtype):
    """RMSNormFunction forward + backward against fp64 autograd of the formula (fp64 inv_rms with its error term)."""
    from d9d_b200.kernel.normalization.rms import rms_norm
    from tests.pointwise_reference import inv_rms_rel

    M, N = 1000, 1024
    x = torch.randn(M, N, device="cuda").to(dtype).requires_grad_()
    w = (torch.randn(N, device="cuda") * 0.1 + 1).to(dtype).requires_grad_()
    dy = torch.randn(M, N, device="cuda").to(dtype)
    out = rms_norm(x, w, EPS)
    out.backward(dy)
    ref, bound, _, _ = rms_norm_fwd_ref(x.detach(), w.detach(), EPS, False)
    check("rms_norm.autograd.out", out.detach(), ref, bound)
    x64, w64 = x.detach().double().requires_grad_(), w.detach().double().requires_grad_()
    (x64 * torch.rsqrt(x64.square().mean(-1, keepdim=True) + float(torch.tensor(EPS, dtype=torch.float32))) * w64).backward(dy.double())
    ir64 = torch.rsqrt(x64.detach().square().mean(-1) + float(torch.tensor(EPS, dtype=torch.float32)))
    dx_ref, dx_b, dw_ref, dw_b = rms_norm_bwd_ref(dy, x.detach(), w.detach(), ir64, False, ir_rel=inv_rms_rel(N))
    torch.testing.assert_close(dx_ref, x64.grad, rtol=1e-9, atol=1e-9)  # the reference is the fp64 autograd gradient
    check("rms_norm.autograd.dx", x.grad, dx_ref, dx_b)
    check("rms_norm.autograd.dw", w.grad, dw_ref, dw_b)


@pytest.mark.parametrize("N", [8, 64, 128, 256, 512, 1024, 2048, 4096, 8192])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("zc", [False, True])
def test_rms_norm_bwd_exact_probe(ops, N, dtype, zc):
    """inv_rms = 1, N a power of two, integer x / dy / w: every product and partial sum is exact in fp32.  dy is non-zero
    only in the first and last rows and on warp, block and pass boundaries, with every column total exact in the output
    dtype, so a dropped or double-counted row, warp or block partial changes a column.

    The backward grid is the resident block count capped at num_sms * 8, and the resident count depends on the kernel's
    registers and shared memory.  So the pass-boundary rows are placed for every grid of b * num_sms blocks, b = 1..8;
    whichever the launcher picks, its boundaries are among them, and M gives the largest grid three passes."""
    per_block, per_pass = _rms_geometry(N, False)
    M = 3 * per_pass + 5
    per_warp = max(1, per_block // 8)
    rows = {0, per_warp - 1, per_warp, per_block - 1, per_block, M - 1}
    for b in range(1, 9):  # a grid of b blocks per SM: one pass covers per_block * b * num_sms rows
        pp = per_block * b * sms()
        rows |= {pp - 1, pp, 2 * pp - 1, 2 * pp, 2 * pp + per_block}
    rows = sorted(r for r in rows if r < M)
    x = (_signs((M, N), torch.float32) * _ints((M, N), 1, 2, torch.float32)).to(dtype)
    w = _ints((N,), -2, 2, torch.float32).to(dtype)
    dy = torch.zeros(M, N, device="cuda", dtype=dtype)
    dy[rows] = _signs((len(rows), N), dtype)
    inv = torch.ones(M, device="cuda")
    dx, dw = ops.rms_norm_bwd(dy, x, w, inv, zc)
    dx_ref, _, dw_ref, _ = rms_norm_bwd_ref(dy, x, w, inv, zc)
    assert torch.equal(dw, dw_ref.to(dtype)), (dw - dw_ref.to(dtype)).abs().max()
    assert torch.equal(dx, dx_ref.to(dtype))


def test_rms_norm_refused_shapes_and_empty(ops):
    x = torch.randn(4, 12, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.rms_norm_fwd(x, torch.ones(12, device="cuda", dtype=torch.bfloat16), EPS, False)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.rms_norm_bwd(x, x, torch.ones(12, device="cuda", dtype=torch.bfloat16), torch.ones(4, device="cuda"), False)
    x = torch.randn(4, 16392, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="N > 16384"):
        ops.rms_norm_fwd(x, torch.ones(16392, device="cuda", dtype=torch.bfloat16), EPS, False)
    x = torch.randn(4, 8200, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="N > 8192"):
        ops.rms_norm_bwd(x, x, torch.ones(8200, device="cuda", dtype=torch.bfloat16), torch.ones(4, device="cuda"), False)
    with pytest.raises(RuntimeError, match="weight"):
        ops.rms_norm_fwd(x[:, :1024].contiguous(), torch.ones(512, device="cuda", dtype=torch.bfloat16), EPS, False)
    # M = 0: nothing to normalise, and the weight gradient is exactly zero
    x0 = torch.empty(0, 1024, device="cuda", dtype=torch.bfloat16)
    w = torch.ones(1024, device="cuda", dtype=torch.bfloat16)
    out, inv = ops.rms_norm_fwd(x0, w, EPS, False)
    assert out.shape == (0, 1024) and inv.shape == (0,)
    for N in (64, 1024, 4096):
        x0 = torch.empty(0, N, device="cuda", dtype=torch.bfloat16)
        dx, dw = ops.rms_norm_bwd(x0, x0, torch.ones(N, device="cuda", dtype=torch.bfloat16), torch.empty(0, device="cuda"), False)
        assert dx.shape == (0, N) and torch.equal(dw, torch.zeros_like(dw))


# ============================================================================ SiLU * mul
def _ew_per_pass() -> int:
    return sms() * 16 * 256  # ew_grid: at most num_sms * 16 blocks of 256 threads, one 8-wide vector each (elementwise.cu:650)


@pytest.mark.parametrize("n", [1, 7, 8, 9, 12345, "persistent"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_silu_mul(ops, n, dtype):
    """The vector loop and the scalar tail (n % 8 elements) both run; the persistent size makes three passes plus 5."""
    if n == "persistent":
        n = 3 * _ew_per_pass() * 8 + 5
    gen = torch.Generator(device="cuda").manual_seed(n)
    x = (torch.randn(n, device="cuda", generator=gen) * 3).to(dtype)
    y = torch.randn(n, device="cuda", generator=gen).to(dtype)
    g = torch.randn(n, device="cuda", generator=gen).to(dtype)
    out = ops.silu_mul_fwd(x, y)
    check("silu_mul_fwd", out, *silu_mul_fwd_ref(x, y))
    dx, dy = ops.silu_mul_bwd(g, x, y)
    dx_ref, dx_b, dy_ref, dy_b = silu_mul_bwd_ref(g, x, y)
    check("silu_mul_bwd.dx", dx, dx_ref, dx_b)
    check("silu_mul_bwd.dy", dy, dy_ref, dy_b)


# ============================================================================ SiLU * mul * probs
def _probs_persistent_rows(cols: int) -> int:
    fwd = _ew_per_pass() * 8 // cols  # silu_mul_probs_fwd: ew_grid over rows * cols / 8 vectors
    bwd = sms() * 8 * 8  # silu_mul_probs_bwd: one warp per row, at most num_sms * 8 blocks (elementwise.cu:748)
    return 3 * max(fwd, bwd) + 5


@pytest.mark.parametrize("cols", [8, 576, 2056])
@pytest.mark.parametrize("rows", [1, 777, "persistent"])
@pytest.mark.parametrize("valid", [None, 0, "mid", "rows", "rows+5"])
def test_silu_mul_probs(ops, cols, rows, valid):
    """Rows below ``valid_rows`` are compared.  Rows at or above it are unspecified by contract (the expert layout never
    reads them) and are not compared."""
    if rows == "persistent":
        rows = _probs_persistent_rows(cols)
    nvalid = {None: rows, 0: 0, "mid": rows // 2 | 1, "rows": rows, "rows+5": rows + 5}[valid]
    vr = None if valid is None else torch.tensor([nvalid], device="cuda", dtype=torch.int32)
    r = min(rows, nvalid)
    gen = torch.Generator(device="cuda").manual_seed(rows * 7 + cols)
    x = (torch.randn(rows, cols, device="cuda", generator=gen) * 3).bfloat16()
    y = torch.randn(rows, cols, device="cuda", generator=gen).bfloat16()
    g = torch.randn(rows, cols, device="cuda", generator=gen).bfloat16()
    p = torch.rand(rows, device="cuda", generator=gen)
    out = ops.silu_mul_probs_fwd(x, y, p, vr)
    check("silu_mul_probs_fwd", out[:r], *silu_mul_probs_fwd_ref(x[:r], y[:r], p[:r]))
    dx, dy, dp = ops.silu_mul_probs_bwd(g, x, y, p, vr)
    dx_ref, dx_b, dy_ref, dy_b, dp_ref, dp_b = silu_mul_probs_bwd_ref(g[:r], x[:r], y[:r], p[:r])
    check("silu_mul_probs_bwd.dx", dx[:r], dx_ref, dx_b)
    check("silu_mul_probs_bwd.dy", dy[:r], dy_ref, dy_b)
    check("silu_mul_probs_bwd.dprobs", dp[:r], dp_ref, dp_b)


@pytest.mark.parametrize("cols", [8, 576, 2056])
def test_silu_mul_probs_dprobs_exact_probe(ops, cols):
    """x in {0, 32}: silu(0) = 0 and silu(32) = 32 exactly in fp32 (exp(-32) vanishes next to 1), so with integer g and y
    each row's dprobs is an exact integer; a row's sum taken from another row or losing a lane shows."""
    rows = _probs_persistent_rows(cols)
    x = (torch.randint(0, 2, (rows, cols), device="cuda") * 32).bfloat16()
    y = _ints((rows, cols), -2, 2, torch.bfloat16)
    g = _ints((rows, cols), -3, 3, torch.bfloat16)
    p = torch.rand(rows, device="cuda")
    _, _, dp = ops.silu_mul_probs_bwd(g, x, y, p)
    ref = (g.double() * x.double() * y.double()).sum(-1)
    assert torch.equal(dp.double(), ref), (dp.double() - ref).abs().max()


# ============================================================================ RoPE
def _rope_cache(maxpos, rope_dim, style, quarter=False, gen=None):
    if quarter:  # quarter turns: cos in {0, +-1}, sin in {0, +-1}, so the rotation is an exact signed permutation
        qt = torch.randint(0, 4, (maxpos, rope_dim // 2), device="cuda", generator=gen)
        c = torch.tensor([1.0, 0.0, -1.0, 0.0], device="cuda")[qt]
        s = torch.tensor([0.0, 1.0, 0.0, -1.0], device="cuda")[qt]
    else:
        ang = torch.rand(maxpos, rope_dim // 2, device="cuda", generator=gen) * 2 * math.pi
        c, s = ang.cos(), ang.sin()
    if style == 0:
        return torch.cat([c, c], -1).contiguous(), torch.cat([s, s], -1).contiguous()
    return c.repeat_interleave(2, -1).contiguous(), s.repeat_interleave(2, -1).contiguous()


def _rope_x(T, H, D, packed, gen):
    if not packed:
        return torch.randn(T, H, D, device="cuda", generator=gen).bfloat16()
    buf = torch.randn(T, 3 * H * D + 2, device="cuda", generator=gen).bfloat16()  # q | k | v, plus a pad: stride > H * D
    return buf[:, H * D: 2 * H * D].unflatten(1, (H, D))


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("i", range(17))
@pytest.mark.parametrize("style", [0, 1])
def test_rope(ops, D, i, style):
    """Every rope_dim the host accepts for D (a multiple of D / 16 up to D), both styles, forward and inverse; x is a slice
    of a packed qkv buffer for odd multiples; positions include 0, max_pos - 1 and repeats."""
    rope_dim = i * D // 16
    T, H, maxpos = 97, 3, 200
    gen = torch.Generator(device="cuda").manual_seed(D * 100 + i * 2 + style)
    x = _rope_x(T, H, D, packed=i % 2 == 1, gen=gen)
    pos = torch.randint(0, maxpos, (T,), device="cuda", generator=gen)
    pos[0], pos[1], pos[2:6] = 0, maxpos - 1, 17
    for quarter in (False, True):
        cos, sin = _rope_cache(maxpos, rope_dim, style, quarter, gen)
        for inverse in (False, True):
            out = ops.rope_apply(x, cos, sin, pos, style, inverse)
            ref, bound = rope_ref(x, cos, sin, pos, style, inverse)
            if quarter:
                assert torch.equal(out, ref.bfloat16()), f"quarter-turn rotation not exact (inverse={inverse})"
            else:
                check("rope", out, ref, bound)


def test_rope_grid_stride_and_refused(ops):
    """T * H > 3 * (num_sms * 16 blocks * 8 warps) (rope_apply's cap, elementwise.cu:988): warps take several (token,
    head) rows.  Odd rope_dim and other shapes outside the kernel's pairing are refused."""
    H, D = 4, 128
    T = (3 * sms() * 16 * 8) // H + 7
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = _rope_x(T, H, D, packed=True, gen=gen)
    maxpos = 4096
    pos = torch.randint(0, maxpos, (T,), device="cuda", generator=gen)
    for style in (0, 1):
        cos, sin = _rope_cache(maxpos, 64, style, gen=gen)
        out = ops.rope_apply(x, cos, sin, pos, style, False)
        check("rope", out, *rope_ref(x, cos, sin, pos, style, False))
    x = torch.randn(8, 2, 64, device="cuda").bfloat16()
    pos = torch.zeros(8, dtype=torch.long, device="cuda")
    for rd in (5, 6, 66):  # odd, not a multiple of D / 16, wider than D
        c = torch.ones(1, rd, device="cuda")
        with pytest.raises(RuntimeError, match="rope"):
            ops.rope_apply(x, c, c, pos, 0, False)


# ============================================================================ fused q/k RMSNorm + RoPE
def _qk_tokens_per_pass() -> int:
    return sms() * 8 * 8  # qk_norm_rope_grid: one warp per token, at most num_sms * 8 blocks (qk_norm_rope.cu:268-269)


def _qk_inputs(T, Hq, Hk, D, rope_dim, style, zc, packed, gen):
    if packed:
        buf = torch.randn(T, (Hq + 2 * Hk) * D, device="cuda", generator=gen).bfloat16()
        q = buf[:, : Hq * D].unflatten(1, (Hq, D))
        k = buf[:, Hq * D: (Hq + Hk) * D].unflatten(1, (Hk, D))
    else:
        q = torch.randn(T, Hq, D, device="cuda", generator=gen).bfloat16()
        k = torch.randn(T, Hk, D, device="cuda", generator=gen).bfloat16()
    if not packed:  # heads of different scale
        q = q * (torch.rand(T, Hq, 1, device="cuda", generator=gen) * 3 + 0.1).bfloat16()
    wq = (torch.randn(D, device="cuda", generator=gen) * 0.1 + (0.0 if zc else 1.0)).bfloat16()
    wk = (torch.randn(D, device="cuda", generator=gen) * 0.1 + (0.0 if zc else 1.0)).bfloat16()
    ang = torch.rand(T, rope_dim // 2, device="cuda", generator=gen) * 2 * math.pi
    ang = torch.cat([ang, ang], -1) if style == 0 else ang.repeat_interleave(2, -1)
    return q, k, wq, wk, ang.cos().contiguous(), ang.sin().contiguous()


def _check_qk(ops, T, Hq, Hk, D, rope_dim, style, zc, packed, through_autograd):
    from d9d_b200.kernel.rope.fused_qk import qk_norm_rope

    gen = torch.Generator(device="cuda").manual_seed(T * 13 + Hq * 7 + Hk + D + rope_dim + style)
    q, k, wq, wk, cos, sin = _qk_inputs(T, Hq, Hk, D, rope_dim, style, zc, packed, gen)
    gq = torch.randn(T, Hq, D, device="cuda", generator=gen).bfloat16()
    gk = torch.randn(T, Hk, D, device="cuda", generator=gen).bfloat16()
    qo, ko, inv = ops.qk_norm_rope_fwd(q, k, wq, wk, cos, sin, EPS, zc, style)
    qo_r, qo_b, ko_r, ko_b, ir_r, ir_b = qk_norm_rope_fwd_ref(q, k, wq, wk, cos, sin, EPS, zc, style, inv_rms=inv)
    check("qk_norm_rope_fwd.inv_rms", inv, ir_r, ir_b)
    check("qk_norm_rope_fwd.q", qo, qo_r, qo_b)
    check("qk_norm_rope_fwd.k", ko, ko_r, ko_b)
    refs = qk_norm_rope_bwd_ref(gq, gk, q, k, wq, wk, cos, sin, inv, zc, style)
    if through_autograd:
        if packed:  # the gradient flows through the packed buffer's views
            base = q._base.detach().clone().requires_grad_()
            lq = base[:, : Hq * D].unflatten(1, (Hq, D))
            lk = base[:, Hq * D: (Hq + Hk) * D].unflatten(1, (Hk, D))
        else:
            lq, lk = q.clone().requires_grad_(), k.clone().requires_grad_()
        lwq, lwk = wq.clone().requires_grad_(), wk.clone().requires_grad_()
        aq, ak = qk_norm_rope(lq, lk, lwq, lwk, cos, sin, EPS, zc, style)
        assert torch.equal(aq, qo) and torch.equal(ak, ko)
        torch.autograd.backward([aq, ak], [gq, gk])
        if packed:
            dq, dk = base.grad[:, : Hq * D].unflatten(1, (Hq, D)), base.grad[:, Hq * D: (Hq + Hk) * D].unflatten(1, (Hk, D))
        else:
            dq, dk = lq.grad, lk.grad
        dwq, dwk = lwq.grad, lwk.grad  # rounded to the weights' bf16
    else:
        dq, dk, dwq, dwk = ops.qk_norm_rope_bwd(gq, gk, q, k, wq, wk, cos, sin, inv, zc, style)
    dq_r, dq_b, dk_r, dk_b, dwq_r, dwq_b, dwk_r, dwk_b = refs
    check("qk_norm_rope_bwd.dq", dq, dq_r, dq_b)
    check("qk_norm_rope_bwd.dk", dk, dk_r, dk_b)
    check("qk_norm_rope_bwd.dwq", dwq, dwq_r, dwq_b + rounding(dwq_r, dwq.dtype))
    check("qk_norm_rope_bwd.dwk", dwk, dwk_r, dwk_b + rounding(dwk_r, dwk.dtype))


# Hq + Hk = 2, 6, 8, 20, 10, 5: every D gets a partly empty last head iteration (5 heads at D = 256, where one iteration
# covers two heads)
QK_HEADS = [(1, 1), (5, 1), (6, 2), (16, 4), (7, 3), (4, 1)]


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("rope_sel", ["16", "32", "D/2", "D"])
@pytest.mark.parametrize("style", [0, 1])
@pytest.mark.parametrize("heads", QK_HEADS)
def test_qk_norm_rope(ops, D, rope_sel, style, heads):
    """Head counts that leave the last head iteration (GROUPS * ROWS_IN_FLIGHT = 8, 4 or 2 heads, qk_norm_rope.cu:106)
    partly empty, at every D; q / k contiguous through the raw ops and as packed-qkv views through the autograd
    function; zero_centered on and off."""
    rope_dim = {"16": 16, "32": 32, "D/2": D // 2, "D": D}[rope_sel]
    if rope_sel == "D/2" and D == 64:
        pytest.skip("rope_dim 32: same case as rope_sel 32")
    Hq, Hk = heads
    for zc, packed in ((False, False), (True, True)):
        _check_qk(ops, 7, Hq, Hk, D, rope_dim, style, zc, packed, through_autograd=packed)


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("style", [0, 1])
@pytest.mark.parametrize("T", [1, "persistent"])
def test_qk_norm_rope_tokens(ops, D, style, T):
    """T = 1 and a persistent T: every warp takes at least three tokens plus a ragged tail, so the per-lane dW
    accumulators carry over from token to token.  7 + 2 heads leave the last head iteration partly empty at every D."""
    if T == "persistent":
        T = 3 * _qk_tokens_per_pass() + 5
    _check_qk(ops, T, 7, 2, D, D // 2, style, True, True, through_autograd=False)
    _check_qk(ops, T, 6, 2, D, 16, style, False, False, through_autograd=False)


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("style", [0, 1])
def test_qk_norm_rope_dw_exact_probe(ops, D, style):
    """inv_rms = 1, quarter-turn angles (the rotation is an exact signed permutation) and integer q, k, w: dwq / dwk are
    exact.  The incoming gradient is non-zero only in the first and last tokens and on block and pass boundaries.  With
    7 + 2 heads the last head iteration is partly empty at every D: its idle rows reload head 0, and adding them to dwq
    would change it."""
    tpp = _qk_tokens_per_pass()
    T, Hq, Hk = 3 * tpp + 5, 7, 2
    toks = sorted({0, 7, 8, tpp - 1, tpp, 2 * tpp - 1, 2 * tpp + 8, 3 * tpp - 1, 3 * tpp, T - 1})
    q = (_signs((T, Hq, D), torch.float32) * _ints((T, Hq, D), 1, 2, torch.float32)).bfloat16()
    k = (_signs((T, Hk, D), torch.float32) * _ints((T, Hk, D), 1, 2, torch.float32)).bfloat16()
    wq, wk = _ints((D,), -2, 2, torch.bfloat16), _ints((D,), -2, 2, torch.bfloat16)
    qt = torch.randint(0, 4, (T, D // 2), device="cuda")
    c = torch.tensor([1.0, 0.0, -1.0, 0.0], device="cuda")[qt]
    s = torch.tensor([0.0, 1.0, 0.0, -1.0], device="cuda")[qt]
    cos = (torch.cat([c, c], -1) if style == 0 else c.repeat_interleave(2, -1)).contiguous()
    sin = (torch.cat([s, s], -1) if style == 0 else s.repeat_interleave(2, -1)).contiguous()
    gq = torch.zeros(T, Hq, D, device="cuda", dtype=torch.bfloat16)
    gk = torch.zeros(T, Hk, D, device="cuda", dtype=torch.bfloat16)
    gq[toks], gk[toks] = _signs((len(toks), Hq, D), torch.bfloat16), _signs((len(toks), Hk, D), torch.bfloat16)
    inv = torch.ones(T, Hq + Hk, device="cuda")
    dq, dk, dwq, dwk = ops.qk_norm_rope_bwd(gq, gk, q, k, wq, wk, cos, sin, inv, False, style)
    dq_r, _, dk_r, _, dwq_r, _, dwk_r, _ = qk_norm_rope_bwd_ref(gq, gk, q, k, wq, wk, cos, sin, inv, False, style)
    assert torch.equal(dwq.double(), dwq_r), (dwq.double() - dwq_r).abs().max()
    assert torch.equal(dwk.double(), dwk_r), (dwk.double() - dwk_r).abs().max()
    assert torch.equal(dq, dq_r.bfloat16()) and torch.equal(dk, dk_r.bfloat16())


def _poison_allocator(numels: list[int]) -> None:
    """Hand NaN-filled blocks of these sizes back to the caching allocator, so an output the kernel never writes is NaN."""
    keep = [torch.full((n,), float("nan"), device="cuda") for n in numels for _ in range(16)]
    del keep


@pytest.mark.parametrize("D", [64, 128, 256])
def test_qk_norm_rope_bwd_no_tokens_zero_weight_grads(ops, D):
    """T = 0 (an empty shard or micro-batch): the weight gradients are exactly zero, not uninitialised memory."""
    Hq, Hk, rope_dim = 4, 2, D
    q = torch.empty(0, Hq, D, device="cuda", dtype=torch.bfloat16)
    k = torch.empty(0, Hk, D, device="cuda", dtype=torch.bfloat16)
    wq = torch.ones(D, device="cuda", dtype=torch.bfloat16)
    wk = torch.ones(D, device="cuda", dtype=torch.bfloat16)
    cos = torch.empty(0, rope_dim, device="cuda")
    sin = torch.empty(0, rope_dim, device="cuda")
    inv = torch.empty(0, Hq + Hk, device="cuda")
    qo, ko, inv0 = ops.qk_norm_rope_fwd(q, k, wq, wk, cos, sin, EPS, False, 0)
    assert qo.shape == (0, Hq, D) and ko.shape == (0, Hk, D) and inv0.shape == (0, Hq + Hk)
    _poison_allocator([D, 2 * D])
    dq, dk, dwq, dwk = ops.qk_norm_rope_bwd(q, k, q, k, wq, wk, cos, sin, inv, False, 0)
    torch.cuda.synchronize()
    assert dq.shape == (0, Hq, D) and dk.shape == (0, Hk, D)
    assert torch.equal(dwq, torch.zeros_like(dwq)), dwq[:8]
    assert torch.equal(dwk, torch.zeros_like(dwk)), dwk[:8]


# ============================================================================ MoE layout / permute / gather
def _layout_ref(ids: torch.Tensor, E: int, align: int):
    """Counts, aligned segment offsets and the row map of a stable sort by expert (CPU)."""
    flat = ids.flatten().cpu()
    valid = (flat >= 0) & (flat < E)
    key = torch.where(valid, flat, torch.full_like(flat, E))
    order = torch.sort(key, stable=True).indices
    counts = torch.bincount(flat[valid], minlength=E)
    seg = torch.zeros(E + 1, dtype=torch.long)
    seg[1:] = ((counts + align - 1) // align * align).cumsum(0)
    row_map = torch.full_like(flat, -1)
    first = torch.zeros(E + 1, dtype=torch.long)
    first[1:] = counts.cumsum(0)
    sk = key[order]
    rank = torch.arange(len(flat)) - first[sk.clamp_max(E - 1)] if E > 0 else torch.zeros(0, dtype=torch.long)
    dst = seg[sk.clamp_max(E - 1)] + rank
    row_map[order[sk < E]] = dst[sk < E]
    return counts, seg, row_map


def _moe_ids(T, k, E, gen, kind):
    if kind == "dropped":
        return torch.full((T, k), -1, dtype=torch.long, device="cuda")
    ids = torch.randint(-2, E + 2, (T, k), device="cuda", generator=gen)  # ids < 0 and >= E are dropped
    ids[1, :] = int(ids[1, 0])  # duplicates within a token
    ids[2, :] = E - 1
    return ids


@pytest.mark.parametrize("E", [1, 2, 1000, 1024])
@pytest.mark.parametrize("k", [1, 8, 32])
@pytest.mark.parametrize("align", [1, 128])
@pytest.mark.parametrize("kind", ["mixed", "dropped"])
def test_moe_layout_permute_gather(ops, E, k, align, kind):
    """T * k spans ~40 chunks of 1024 entries (five blocks of eight chunk-warps, moe.cu:14, 217); every row_map entry
    against a stable CPU sort; capacity exactly the aligned total and larger."""
    T = 40_000 // k + 3
    H = 264
    gen = torch.Generator(device="cuda").manual_seed(E * 100 + k + align)
    ids = _moe_ids(T, k, E, gen, kind)
    counts_r, seg_r, rm_r = _layout_ref(ids, E, align)
    total = int(seg_r[-1])
    for cap in (total, total + (256 if align == 128 else 37)):
        counts, seg, row_map, tile_group = ops.moe_build_layout(ids, E, align, cap)
        assert torch.equal(counts.long().cpu(), counts_r)
        assert torch.equal(seg.long().cpu(), seg_r)
        assert torch.equal(row_map.long().cpu(), rm_r)
        if align == 128:  # the compact layout (align = 1) has no tile table
            starts = torch.arange(cap // 128) * 128
            owner = torch.searchsorted(seg_r[1:], starts, right=True)
            assert torch.equal(tile_group.long().cpu(), torch.where(starts < total, owner, -1))

    rm = rm_r.cuda()
    valid = rm >= 0
    tok = torch.arange(T, device="cuda").repeat_interleave(k)
    x = torch.randn(T, H, device="cuda", generator=gen).bfloat16()
    probs = torch.rand(T, k, device="cuda", generator=gen)
    xp, pp = ops.moe_permute(x, probs, row_map, counts, seg, cap)
    assert torch.equal(xp[rm[valid]], x[tok[valid]])
    assert torch.equal(pp[rm[valid]], probs.flatten()[valid])
    pad = torch.ones(cap, dtype=torch.bool, device="cuda")
    pad[rm[valid]] = False
    pad[total:] = False  # rows past the last segment are left untouched
    assert (xp[pad] == 0).all() and (pp[pad] == 0).all()

    yp = torch.randn(cap, H, device="cuda", generator=gen).bfloat16()
    dpp = torch.randn(cap, device="cuda", generator=gen)
    y, dprobs = ops.moe_gather(yp, dpp, row_map, T, k)
    y_r, y_b, dp_r = moe_gather_ref(yp, row_map, T, k, dpp)
    check("moe_gather", y, y_r, y_b)
    assert torch.equal(dprobs.double(), dp_r)
    y2, _ = ops.moe_gather(yp, None, row_map, T, k)
    assert torch.equal(y2, y)
    # exact probe: integer rows, so every sum of k rows is exact; a dropped or doubled row changes it
    ypi = _ints((cap, H), -4, 4, torch.bfloat16)
    yi, _ = ops.moe_gather(ypi, None, row_map, T, k)
    assert torch.equal(yi.double(), moe_gather_ref(ypi, row_map, T, k)[0])


def test_moe_zero_pad(ops):
    """Called directly: the pad rows [seg[e] + counts[e], seg[e + 1]) are zeroed and nothing else is written."""
    E, H = 7, 136
    counts = torch.tensor([0, 1, 127, 128, 129, 5, 300], dtype=torch.int32)
    seg = torch.zeros(E + 1, dtype=torch.int32)
    seg[1:] = ((counts + 127) // 128 * 128).cumsum(0)
    cap = int(seg[-1]) + 128
    xp = torch.full((cap, H), 7.0, device="cuda", dtype=torch.bfloat16)
    pp = torch.full((cap,), 7.0, device="cuda")
    ops.moe_zero_pad(xp, pp, counts.cuda(), seg.cuda())
    pad = torch.zeros(cap, dtype=torch.bool)
    for e in range(E):
        pad[int(seg[e]) + int(counts[e]): int(seg[e + 1])] = True
    pad = pad.cuda()
    assert (xp[pad] == 0).all() and (pp[pad] == 0).all()
    assert (xp[~pad] == 7).all() and (pp[~pad] == 7).all()


# ============================================================================ sumsq_accumulate / scale_inplace
@pytest.mark.parametrize("n", [1, 7, 8, 9, 12345, "persistent"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_sumsq_accumulate_and_scale(ops, n, dtype):
    """``out += sum(x^2)`` into a non-zero ``out``; block count from sumsq_accumulate's cap (num_sms * 4,
    elementwise.cu:1054) and ew_grid's (num_sms * 16) for scale_inplace_."""
    cap = sms() * 4
    if n == "persistent":
        n = 3 * _ew_per_pass() * 8 + 5
    blocks = max(1, min(cap, ((n >> 3) + 255) // 256))
    x = torch.randn(n, device="cuda").to(dtype)
    out0 = float(n)
    out = torch.tensor([out0], device="cuda")
    ops.sumsq_accumulate_(x, out)
    ref, bound = sumsq_ref(x, out0, adds=blocks)
    err = abs(float(out) - ref)
    assert err <= bound, (float(out), ref, bound)
    WORST["sumsq_accumulate"] = max(WORST.get("sumsq_accumulate", 0.0), err / bound)
    # exact probe: sparse integers, every partial exact; a lost or doubled block / tail element shows
    xi = torch.zeros(n, device="cuda", dtype=dtype)
    xi[torch.randint(0, n, (min(n, 4096),), device="cuda")] = _ints((min(n, 4096),), 1, 3, dtype)
    xi[0], xi[-1] = 2, 3
    out = torch.tensor([1024.0], device="cuda")
    ops.sumsq_accumulate_(xi, out)
    assert float(out) == 1024.0 + float(xi.double().square().sum())
    sc = torch.tensor([0.7], device="cuda")
    y = x.clone()
    ops.scale_inplace_(y, sc)
    ref = x.double() * float(sc)
    check("scale_inplace", y, ref, U32 * ref.abs() + rounding(ref, dtype))


# ============================================================================ 16-byte alignment
def _offset_view(t: torch.Tensor, off: int = 3) -> torch.Tensor:
    """A contiguous copy of t that starts `off` elements past a 16-byte boundary."""
    flat = torch.empty(t.numel() + 16, device=t.device, dtype=t.dtype)
    v = flat[off: off + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0
    return v


def test_unaligned_operands_refused(ops):
    """Offset views pass is_contiguous() but not the 16-byte vector accesses: the host refuses them before any launch."""
    x = torch.randn(64, 256, device="cuda").bfloat16()
    w = torch.ones(256, device="cuda", dtype=torch.bfloat16)
    inv = torch.ones(64, device="cuda")
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.rms_norm_fwd(_offset_view(x), w, EPS, False)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.rms_norm_fwd(x, _offset_view(w), EPS, False)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.rms_norm_bwd(_offset_view(x), x, w, inv, False)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.silu_mul_fwd(_offset_view(x), x)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.silu_mul_bwd(x, x, _offset_view(x))
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.silu_mul_probs_fwd(_offset_view(x), x, inv)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.silu_mul_probs_bwd(x, _offset_view(x), x, inv)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.sumsq_accumulate_(_offset_view(x), torch.zeros(1, device="cuda"))
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.scale_inplace_(_offset_view(x), torch.ones(1, device="cuda"))
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.moe_gather(_offset_view(x), None, torch.zeros(64, dtype=torch.int32, device="cuda"), 64, 1)
    ids = torch.zeros(64, 1, dtype=torch.long, device="cuda")
    counts, seg, row_map, _ = ops.moe_build_layout(ids, 1, 128, 128)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.moe_permute(_offset_view(x), None, row_map, counts, seg, 128)
    q = torch.randn(8, 2, 64, device="cuda").bfloat16()
    wq = torch.ones(64, device="cuda", dtype=torch.bfloat16)
    cs = torch.ones(8, 64, device="cuda")
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.qk_norm_rope_fwd(_offset_view(q, 4), q, wq, wq, cs, cs, EPS, False, 0)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.qk_norm_rope_fwd(q, q, wq, _offset_view(wq), cs, cs, EPS, False, 0)
    with pytest.raises(RuntimeError, match="16-byte"):
        ops.qk_norm_rope_bwd(_offset_view(q, 4), q, q, q, wq, wq, cs, cs, torch.ones(8, 4, device="cuda"), False, 0)
    with pytest.raises(RuntimeError, match="weights"):
        ops.qk_norm_rope_fwd(q, q, wq[:32].contiguous(), wq, cs, cs, EPS, False, 0)


def test_wrappers_copy_unaligned_operands(ops):
    """The Python wrappers copy an offset view into a fresh buffer: the result equals the contiguous-input result."""
    from d9d_b200.kernel.normalization.rms import rms_norm
    from d9d_b200.kernel.rope.fused_qk import qk_norm_rope
    from d9d_b200.kernel.swiglu import silu_mul, silu_mul_probs

    x = torch.randn(33, 520, device="cuda").bfloat16()
    y = torch.randn(33, 520, device="cuda").bfloat16()
    w = (torch.randn(520, device="cuda") * 0.1 + 1).bfloat16()
    p = torch.rand(33, device="cuda")
    assert torch.equal(silu_mul(_offset_view(x), _offset_view(y)), silu_mul(x, y))
    assert torch.equal(silu_mul_probs(_offset_view(x), y, p), silu_mul_probs(x, y, p))
    assert torch.equal(rms_norm(_offset_view(x), _offset_view(w)), rms_norm(x, w))
    xa, xb = _offset_view(x).requires_grad_(), x.clone().requires_grad_()
    g = torch.randn_like(x)
    rms_norm(xa, w).backward(_offset_view(g))
    rms_norm(xb, w).backward(g)
    assert torch.equal(xa.grad, xb.grad)
    T, Hq, Hk, D = 9, 3, 1, 128
    q = torch.randn(T, Hq, D, device="cuda").bfloat16()
    k = torch.randn(T, Hk, D, device="cuda").bfloat16()
    wq = (torch.randn(D, device="cuda") * 0.1 + 1).bfloat16()
    cos, sin = torch.rand(T, 64, device="cuda"), torch.rand(T, 64, device="cuda")
    ref = qk_norm_rope(q, k, wq, wq, cos, sin, EPS, False, 0)
    got = qk_norm_rope(_offset_view(q), _offset_view(k, 5), _offset_view(wq), wq, cos, sin, EPS, False, 0)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
