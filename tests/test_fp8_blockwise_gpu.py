"""Blockwise fp8 on the H100: the 1x128 / 128-token / 128x128 quantisers against their PyTorch emulations, the BLOCKWISE
e4m3 GEMM against an fp64 product of the operands and scales it consumed (per element within a promoted-accumulation
bound, and norm-wise for a long fp32 weight gradient), operand checks, and ``fp8_linear(recipe="blockwise")`` against its
CPU emulation and against fp64."""

import math

import pytest
import torch

from d9d_b200.kernel import fp8

pytestmark = pytest.mark.gpu

U_CHAIN = 2.0**-13  # assumed unit roundoff of the tensor core's e4m3 accumulation inside one 128-deep k-block
U_F32 = 2.0**-24
U_BF16 = 2.0**-8
CANARY = 7.0


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _mismatch_ok(q, qr):
    # the kernels multiply by a fast-math reciprocal of the scale, the emulations divide: at most one e4m3 step apart,
    # and only rarely.  Same-sign e4m3 codes are ordered like their magnitudes, so one step is a code difference of 1
    # (also among subnormals, whose steps are large relative to the value).
    a, b = q.cpu().view(torch.uint8).int(), qr.cpu().view(torch.uint8).int()
    diff = a != b
    if diff.any():
        assert bool(((a[diff] ^ b[diff]) & 0x80 == 0).all()) and int((a[diff] - b[diff]).abs().max()) <= 1
    return float(diff.float().mean())


def _check_scales(s, sr, groups, rows):
    assert s.shape == (groups, rows) and s.stride(1) == 1 and s.stride(0) == (rows + 127) // 128 * 128
    torch.testing.assert_close(s.cpu(), sr, rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------ quantisers
@pytest.mark.parametrize("M,K", [(1000, 576), (256, 7168), (3, 16), (130, 400)])
def test_row_group_quantiser(ops, M, K):
    x = (torch.randn(M, K, device="cuda") * torch.logspace(-2, 2, K, device="cuda")[None]).bfloat16()
    x[M // 2] = 0
    q, s = ops.quantize_blockwise(x)
    qr, sr = fp8.quantize_blockwise_reference(x.cpu())
    assert q.shape == (M, K) and q.dtype == fp8.FP8
    _check_scales(s, sr, (K + 127) // 128, M)
    assert _mismatch_ok(q, qr) < 0.02


@pytest.mark.parametrize("M,C", [(1000, 576), (130, 144), (16384, 64), (5, 32)])
def test_token_group_quantiser(ops, M, C):
    x = (torch.randn(M, C, device="cuda") * torch.logspace(-2, 2, M, device="cuda")[:, None]).bfloat16()
    x[:, 3] = 0
    qt, s = ops.quantize_blockwise_t(x)
    qr, sr = fp8.quantize_blockwise_t_reference(x.cpu())
    pitch = (M + 15) // 16 * 16
    assert qt.shape == (C, M) and qt.stride() == (pitch, 1)
    _check_scales(s, sr, (M + 127) // 128, C)
    assert _mismatch_ok(qt, qr) < 0.02
    full = qt.as_strided((C, pitch), (pitch, 1))
    assert not full[:, M:].float().any()  # the 16-byte row pitch's pad columns are zeros


@pytest.mark.parametrize("N,K", [(576, 7168), (144, 400), (7168, 576)])
def test_weight_block_quantiser_and_its_transposed_copy(ops, N, K):
    w = (torch.randn(N, K, device="cuda") * torch.logspace(-2, 1, N, device="cuda")[:, None]).bfloat16()
    q, s = ops.quantize_weight_blocks(w)
    qt, st = ops.quantize_weight_blocks(w, True)
    qr, sr = fp8.quantize_weight_blocks_reference(w.cpu())
    qtr, str_ = fp8.quantize_weight_blocks_reference(w.cpu(), transpose=True)
    _check_scales(s, sr, (K + 127) // 128, N)
    _check_scales(st, str_, (N + 127) // 128, K)
    assert _mismatch_ok(q, qr) < 0.02 and _mismatch_ok(qt, qtr) < 0.02
    assert torch.equal(qt.view(torch.uint8), q.view(torch.uint8).t())


# ------------------------------------------------------------------------------------------ GEMM
def _exact(aq, sa, bq, sb):
    """fp64 product of what the kernel consumed, and sum_k |a_k b_k| (scaled) for the bound."""
    K = aq.shape[1]
    out = torch.zeros(aq.shape[0], bq.shape[0], dtype=torch.float64, device=aq.device)
    absd = torch.zeros_like(out)
    for kb in range((K + 127) // 128):
        ks = slice(kb * 128, min(K, kb * 128 + 128))
        a = aq[:, ks].double() * sa[kb].double()[:, None]
        b = bq[:, ks].double() * sb[kb].double()[:, None]
        out += a @ b.t()
        absd += a.abs() @ b.abs().t()
    return out, absd


def _bound(absd, k_blocks):
    """Per-element bound on |D - exact| from the accumulation: in-chain accumulation at U_CHAIN per 128-deep k-block, fp32
    for the scaling and across k-blocks.  Callers add the output rounding."""
    return 128 * U_CHAIN * absd + (k_blocks + 3) * U_F32 * absd


def _canaried(M, N, dtype):
    """A [M, N] output inside a larger buffer filled with a canary: 1 row and 8 columns around it."""
    big = torch.full((M + 2, N + 16), CANARY, device="cuda", dtype=dtype)
    return big, big[1 : M + 1, 8 : N + 8]


@pytest.mark.parametrize("M,N,K", [(1000, 576, 7168), (130, 144, 208), (256, 272, 1040), (7, 16, 16), (8192, 576, 576)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_blockwise_gemm_against_fp64(ops, M, N, K, dtype):
    a = torch.randn(M, K, device="cuda").bfloat16()
    a[0, :40] *= 2.0**10  # an outlier group
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    aq, sa = ops.quantize_blockwise(a)
    bq, sb = ops.quantize_weight_blocks(w)
    big, d = _canaried(M, N, dtype)
    ops.gemm_fp8_blockwise(aq, sa, bq, sb, d)
    exact, absd = _exact(aq, sa, bq, sb)
    bound = _bound(absd, math.ceil(K / 128)) + (U_BF16 * exact.abs() if dtype == torch.bfloat16 else U_F32 * exact.abs()) + 1e-30
    ratio = float(((d.double() - exact).abs() / bound).max())
    print(f"blockwise M={M} N={N} K={K} {dtype}: worst err / bound = {ratio:.3f}")
    assert ratio <= 1.0
    outside = torch.ones_like(big, dtype=torch.bool)
    outside[1 : M + 1, 8 : N + 8] = False
    assert bool((big[outside] == CANARY).all())  # no stray writes
    d2 = torch.empty_like(d)
    ops.gemm_fp8_blockwise(aq, sa, bq, sb, d2)
    assert torch.equal(d, d2)  # bitwise reproducible


def test_long_weight_gradient_error_is_that_of_promoted_accumulation(ops):
    """Norm-wise error of an fp32 weight gradient over 16 384 tokens against fp64 of the consumed operands.  Random
    inputs, round-to-nearest at U_CHAIN inside a chain: promoted accumulation gives rel ~= U_CHAIN * sqrt(129 / 6)
    (independent of the token count), one chain over all k tokens U_CHAIN * sqrt((k + 1) / 6), 11x more here."""
    T, out_f, in_f = 16384, 576, 1536
    x = torch.randn(T, in_f, device="cuda").bfloat16()
    dy = torch.randn(T, out_f, device="cuda").bfloat16()
    dyq, sdy = ops.quantize_blockwise_t(dy)
    xq, sx = ops.quantize_blockwise_t(x)
    dw = torch.empty(out_f, in_f, device="cuda")
    ops.gemm_fp8_blockwise(dyq, sdy, xq, sx, dw)
    exact, _ = _exact(dyq, sdy, xq, sx)
    rel = _rel(dw, exact)
    promoted, one_chain = U_CHAIN * math.sqrt(129 / 6), U_CHAIN * math.sqrt((T + 1) / 6)
    print(f"blockwise wgrad {T} tokens: rel err {rel:.2e}; model: promoted {promoted:.2e}, one chain {one_chain:.2e}")
    assert rel <= 3 * promoted


def test_blockwise_ops_refuse_bad_operands(ops):
    M, N, K = 200, 144, 256
    a = torch.randn(M, K, device="cuda").bfloat16()
    w = torch.randn(N, K, device="cuda").bfloat16()
    aq, sa = ops.quantize_blockwise(a)
    bq, sb = ops.quantize_weight_blocks(w)
    d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    bad = [
        (a, sa, bq, sb, d),  # bf16 a
        (aq, sa.contiguous(), bq, sb, d),  # scale rows not padded to 128 (M = 200)
        (aq, sa[:1], bq, sb, d),  # too few k-blocks
        (aq, sa.float().cpu(), bq, sb, d),  # scales on the host
        (aq, sa, bq[:, :128], sb, d),  # K mismatch
        (aq, sa, bq, sb, torch.empty(M, N, device="cuda", dtype=torch.float16)),  # fp16 output
        (aq, sa, bq, sb, torch.empty(M, N + 8, device="cuda", dtype=torch.bfloat16)[:, 1 : N + 1]),  # misaligned output
        (aq, sa, bq, sb, torch.empty(M + 1, N, device="cuda", dtype=torch.bfloat16)),  # wrong output shape
        (aq, sa.narrow(1, 0, M - 1), bq, sb, d),  # scale rows do not match M
    ]
    for args in bad:
        with pytest.raises(RuntimeError):
            ops.gemm_fp8_blockwise(*args)
    with pytest.raises(RuntimeError):
        ops.quantize_blockwise(torch.randn(M, 40, device="cuda").bfloat16())  # K not a multiple of 16
    with pytest.raises(RuntimeError):
        ops.quantize_blockwise_t(torch.randn(M, K, device="cuda"))  # fp32 input
    with pytest.raises(RuntimeError):
        ops.quantize_weight_blocks(torch.randn(100, K, device="cuda").bfloat16())  # N not a multiple of 16
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ layer
@pytest.mark.parametrize("T,in_f,out_f", [(1000, 576, 1536), (2048, 7168, 576), (130, 144, 272)])
@pytest.mark.parametrize("grad_fp32", [False, True])
def test_blockwise_linear_against_emulation_and_fp64(T, in_f, out_f, grad_fp32):
    torch.manual_seed(T + in_f)
    x = torch.randn(T, in_f, device="cuda").bfloat16()
    w = (torch.randn(out_f, in_f, device="cuda") * in_f**-0.5).bfloat16()
    g = torch.randn(T, out_f, device="cuda").bfloat16()
    xg, wg = x.clone().requires_grad_(), w.clone().requires_grad_()
    if grad_fp32:
        wg.grad_dtype = torch.float32
    y = fp8.fp8_linear(xg, wg, recipe="blockwise")
    y.backward(g)
    assert y.dtype == torch.bfloat16 and wg.grad.dtype == (torch.float32 if grad_fp32 else torch.bfloat16)
    # the same recipe emulated on the CPU
    xc, wc = x.cpu().requires_grad_(), w.cpu().requires_grad_()
    yc = fp8.fp8_linear(xc, wc, recipe="blockwise")
    yc.backward(g.cpu())
    assert _rel(y.cpu(), yc) < 2e-2 and _rel(xg.grad.cpu(), xc.grad) < 2e-2 and _rel(wg.grad.cpu(), wc.grad) < 2e-2
    # and against fp64 of the bf16 inputs
    xd, wd = x.double().requires_grad_(), w.double().requires_grad_()
    yd = xd @ wd.t()
    yd.backward(g.double())
    errs = (_rel(y, yd), _rel(xg.grad, xd.grad), _rel(wg.grad, wd.grad))
    print(f"blockwise linear T={T} {in_f}->{out_f}: rel err y / dx / dW = {errs[0]:.2e} / {errs[1]:.2e} / {errs[2]:.2e}")
    assert max(errs) < 0.06
