"""FP8 wgmma kernels (e4m3 with epilogue scales, MXFP8 block scales) and their quantisers against their PyTorch
emulations, norm-wise.  The per-element checks against fp64 models are in ``test_fp8_kernels_gpu.py``."""

import pytest
import torch

from d9d_b200.kernel import fp8

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.mark.parametrize("M,K", [(256, 256), (1000, 528), (4096, 768)])
def test_quantize_rowwise(ops, M, K):
    x = (torch.randn(M, K, device="cuda") * torch.logspace(-2, 2, M, device="cuda")[:, None]).bfloat16()
    x[5] = 0
    q, s = ops.quantize_rowwise(x)
    qr, sr = fp8.quantize_rowwise_reference(x)
    assert torch.allclose(s, sr, rtol=1e-6, atol=0)
    # the kernel multiplies by a fast-math 1/s: at most one e4m3 step away from the division-based reference, and only
    # rarely (the exact admissible-code check is in test_fp8_kernels_gpu.py)
    assert (q.float() != qr.float()).float().mean().item() < 0.02
    assert _rel(q.float() * s[:, None], x) < 0.04


@pytest.mark.parametrize("R,C", [(256, 256), (1000, 520), (777, 96)])
def test_quantize_colwise_transposed(ops, R, C):
    x = (torch.randn(R, C, device="cuda") * torch.logspace(-2, 2, C, device="cuda")[None]).bfloat16()
    qt, s = ops.quantize_colwise_t(x)
    assert qt.shape == (C, R) and qt.stride(1) == 1 and qt.stride(0) % 16 == 0
    qr, sr = fp8.quantize_colwise_t_reference(x)
    assert torch.allclose(s, sr, rtol=1e-6, atol=0)
    assert (qt.float() != qr.float()).float().mean().item() < 0.02
    assert _rel((qt.float() * s[:, None]).t(), x) < 0.04


@pytest.mark.parametrize("M,K", [(256, 256), (1000, 512), (300, 1024)])
def test_quantize_mx(ops, M, K):
    x = (torch.randn(M, K, device="cuda") * torch.logspace(-3, 3, K // 32, device="cuda").repeat_interleave(32)[None]).bfloat16()
    x[7, 32:64] = 0
    q, sf = ops.quantize_mx(x)
    qr, er = fp8.quantize_mx_reference(x)
    e = fp8.unpack_mx_scales(sf, M, K)
    assert torch.equal(e, er)
    assert torch.equal(q.float(), qr.float())


@pytest.mark.parametrize("M,N,K", [(256, 256, 256), (1000, 776, 528), (4096, 2048, 768), (333, 128, 256), (128, 64, 128)])
@pytest.mark.parametrize("scales", ["both", "none"])
def test_gemm_fp8_rowcol(ops, M, N, K, scales):
    a = torch.randn(M, K, device="cuda").bfloat16()
    b = torch.randn(N, K, device="cuda").bfloat16()
    aq, sa = ops.quantize_rowwise(a)
    bq, sb = ops.quantize_rowwise(b)
    d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    if scales == "both":
        ops.gemm_fp8(aq, bq, sa, sb, 1.0, d)
        ref = (aq.float() @ bq.float().t()) * sa[:, None] * sb[None, :]
    else:
        ops.gemm_fp8(aq, bq, None, None, 0.5, d)
        ref = (aq.float() @ bq.float().t()) * 0.5
    # one reduced-precision tensor-core chain over K (about 2^-13 per addition, unpromoted) and the bf16 output rounding
    assert _rel(d, ref) < 5e-3
    if scales == "both":
        assert _rel(d, a.float() @ b.float().t()) < 0.06  # end-to-end quantisation error of the recipe


@pytest.mark.parametrize("M,N,K", [(256, 256, 256), (1000, 776, 512), (4096, 2048, 768), (333, 128, 256)])
def test_gemm_mxfp8(ops, M, N, K):
    a = (torch.randn(M, K, device="cuda") * torch.logspace(-1, 1, K // 32, device="cuda").repeat_interleave(32)[None]).bfloat16()
    b = torch.randn(N, K, device="cuda").bfloat16()
    aq, sfa = ops.quantize_mx(a)
    bq, sfb = ops.quantize_mx(b)
    d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm_mxfp8(aq, sfa, bq, sfb, d)
    ref = fp8.dequantize_mx(aq, fp8.unpack_mx_scales(sfa, M, K)) @ fp8.dequantize_mx(bq, fp8.unpack_mx_scales(sfb, N, K)).t()
    assert _rel(d, ref) < 5e-3
    assert _rel(d, a.float() @ b.float().t()) < 0.06


def test_fp8_linear_function_matches_emulation():
    torch.manual_seed(0)
    x = torch.randn(4, 256, 512, device="cuda").bfloat16().requires_grad_()
    w = (torch.randn(1024, 512, device="cuda") * 0.05).bfloat16().requires_grad_()
    y = fp8.fp8_linear(x, w)
    g = torch.randn_like(y)
    y.backward(g)
    xc, wc = x.detach().cpu().requires_grad_(), w.detach().cpu().requires_grad_()
    yc = fp8.fp8_linear(xc, wc)
    yc.backward(g.cpu())
    assert _rel(y.cpu(), yc) < 2e-2
    assert _rel(x.grad.cpu(), xc.grad) < 2e-2
    assert _rel(w.grad.cpu(), wc.grad) < 2e-2
    ref = x.detach().float() @ w.detach().float().t()
    assert _rel(y, ref) < 0.06

