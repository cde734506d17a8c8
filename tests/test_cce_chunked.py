"""Host logic of the fused linear-CE (vocabulary chunk plan, split classifier blocks, accumulation flags) exercised on
CPU through PyTorch stand-ins of the native ops; the kernels themselves are checked in ``test_ops_gpu.py``."""

import pytest
import torch

from d9d_b200.kernel.cce import main as cce
from d9d_b200.kernel.cce.main import linear_cross_entropy, linear_cross_entropy_reference, plan_vocab_chunks


def _problem(T=96, K=32, sizes=(700, 24), seed=0):
    g = torch.Generator().manual_seed(seed)
    e = (torch.randn(T, K, generator=g) * 0.5).requires_grad_()
    ws = [(torch.randn(s, K, generator=g) * 0.2).requires_grad_() for s in sizes]
    tgt = torch.randint(0, sum(sizes), (T,), generator=g)
    tgt[::5] = -100
    tgt[1] = sum(sizes) - 1  # a target inside the last (tiny) block
    return e, ws, tgt


@pytest.mark.parametrize("sizes", [(700,), (700, 24), (300, 260, 8)])
@pytest.mark.parametrize("budget", [1 << 30, 96 * 256 * 2 + 96 * 32 * 4])
@pytest.mark.parametrize("softcap,with_bias", [(None, False), (5.0, True)])
def test_chunked_backward_matches_autograd(monkeypatch, sizes, budget, softcap, with_bias):
    monkeypatch.setattr(cce, "_CHUNK_BYTES", budget)
    e, ws, tgt = _problem(sizes=sizes)
    bias = (torch.randn(sum(sizes)) * 0.3).requires_grad_() if with_bias else None
    loss, lse = linear_cross_entropy(e, ws, tgt, bias=bias, softcap=softcap, reduction="sum", return_lse=True, _emulate=True)
    loss.backward()
    got = [e.grad.clone(), *[w.grad.clone() for w in ws]] + ([bias.grad.clone()] if with_bias else [])

    e2 = e.detach().clone().requires_grad_()
    ws2 = [w.detach().clone().requires_grad_() for w in ws]
    b2 = bias.detach().clone().requires_grad_() if with_bias else None
    nll, lse_ref = linear_cross_entropy_reference(e2, torch.cat(ws2), tgt, b2, -100, softcap)
    nll.sum().backward()
    ref = [e2.grad, *[w.grad for w in ws2]] + ([b2.grad] if with_bias else [])
    assert torch.allclose(loss, nll.sum(), rtol=1e-4, atol=1e-4)
    assert torch.allclose(lse, lse_ref, rtol=1e-4, atol=1e-4)
    for a, b in zip(got, ref):
        # the emulated dlogits buffer is bf16 like the real one
        assert (a - b).norm() / (b.norm() + 1e-9) < 1e-2


def test_plan_respects_budget_and_covers_vocabulary():
    for sizes, T, K in [((151643, 26), 16384, 768), ((151669,), 16384, 2048), ((128256,), 32768, 4096), ((1000, 24), 512, 256)]:
        budget = 256 << 20
        chunks, width, multi = plan_vocab_chunks(sizes, T, K, budget, 132)
        assert T * width * 2 <= max(budget, T * 256 * 2)
        for i, size in enumerate(sizes):
            mine = sorted((r0, r1) for s, r0, r1 in chunks if s == i)
            assert mine[0][0] == 0 and mine[-1][1] == size
            assert all(a[1] == b[0] for a, b in zip(mine, mine[1:]))
            assert all(r1 - r0 <= width for r0, r1 in mine)
        assert multi == (len(chunks) > 1)
    # the flagship problem stays within a few dozen chunks whose dC GEMM fills the 132 SMs of an H100
    chunks, width, _ = plan_vocab_chunks((151643, 26), 16384, 768, 256 << 20, 132)
    assert len(chunks) <= 32 and (width // 128) * 3 <= 132
