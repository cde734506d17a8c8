"""CTA-pair (two-CTA clusters with B multicast, 256-row tiles) variants of the dense GEMM and of the fused linear-CE GEMMs against fp32
PyTorch references - the same checks the single-CTA kernels pass in ``test_ops_gpu.py``."""

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 512, 128), (1000, 776, 520), (4096, 2048, 768), (333, 129 * 8, 72), (8192, 576, 768),
                                   (16384, 128, 768), (2048, 4096, 4096)])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_pair_gemm_nt(ops, M, N, K, out_dtype):
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    d = torch.empty(M, N, device="cuda", dtype=out_dtype)
    ops.gemm(a, b, d, False, False, False, 2)
    assert _rel_err(d, a.float() @ b.float().t()) < (1e-2 if out_dtype == torch.bfloat16 else 1e-4)


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (1000, 776, 520), (4096, 768, 2048)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_pair_gemm_dgrad_layout(ops, M, N, K, accumulate):
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    d0 = torch.randn(M, N, device="cuda", dtype=torch.float32)
    d = d0.clone()
    ops.gemm(a, b, d, False, True, accumulate, 2)
    assert _rel_err(d, a.float() @ b.float() + (d0 if accumulate else 0)) < 1e-4


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (776, 520, 1000), (768, 2048, 4096), (576, 768, 16384)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_pair_gemm_wgrad_layout(ops, M, N, K, accumulate):
    a = torch.randn(K, M, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    d0 = torch.randn(M, N, device="cuda", dtype=torch.float32)
    d = d0.clone()
    ops.gemm(a, b, d, True, True, accumulate, 2)  # accumulate also exercises split-K over CTA pairs
    assert _rel_err(d, a.float().t() @ b.float() + (d0 if accumulate else 0)) < 1e-4


def test_pair_gemm_mn_a_k_b(ops):
    M, N, K = 640, 384, 512
    a = torch.randn(K, M, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, b, d, True, False, False, 2)
    assert _rel_err(d, a.float().t() @ b.float().t()) < 1e-2


def test_pair_gemm_many_tiles_per_pair(ops):
    # more tiles than CTA pairs: every pair walks several tiles through both accumulator stages and all smem stages
    M, N, K = 8192, 8192, 1024
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, b, d, False, False, False, 2)
    ref = torch.empty_like(d)
    ops.gemm(a, b, ref, False, False, False, 1)
    assert torch.equal(d, ref)  # same MMA shape in K and the same accumulation order per element


@pytest.mark.parametrize("T,V,K", [(1024, 5000, 256), (2048, 32000, 768)])
def test_pair_linear_ce(ops, T, V, K):
    prev = ops.gemm_set_pair_mode(1)
    try:
        h = (torch.randn(T, K, device="cuda") * 0.5).bfloat16()
        w = (torch.randn(V, K, device="cuda") * 0.1).bfloat16()
        tgt = torch.randint(0, V, (T,), device="cuda")
        tgt[::7] = -100
        nll, lse = ops.ce_forward(h, w, tgt, -100)
        logits = h.float() @ w.float().t()
        ref = torch.nn.functional.cross_entropy(logits, tgt, ignore_index=-100, reduction="none")
        assert torch.allclose(nll, ref, atol=2e-3, rtol=2e-3)
        assert torch.allclose(lse, torch.logsumexp(logits, -1), atol=2e-3, rtol=2e-3)
        g = torch.rand(T, device="cuda")
        out = torch.empty(T, V, device="cuda", dtype=torch.bfloat16)
        ops.ce_dlogits(h, w, tgt, lse, g, out, -100)
        p = torch.softmax(logits, -1)
        onehot = torch.zeros_like(p)
        valid = tgt != -100
        onehot[valid, tgt[valid]] = 1
        assert _rel_err(out, (p - onehot) * (g * valid)[:, None]) < 2e-2
    finally:
        ops.gemm_set_pair_mode(prev)
