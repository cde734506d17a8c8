"""MXFP8 recipe of ``Fp8Linear`` (forward, dgrad and wgrad quantised along their own reduction dimensions) on the GPU against
its CPU emulation and against fp64."""

import pytest
import torch

from d9d_b200.kernel import fp8

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def test_mxfp8_linear_function_matches_emulation():
    torch.manual_seed(0)
    x = torch.randn(4, 256, 512, device="cuda").bfloat16().requires_grad_()  # 1024 tokens
    w = (torch.randn(1024, 512, device="cuda") * 0.05).bfloat16().requires_grad_()
    y = fp8.fp8_linear(x, w, recipe="mx")
    g = torch.randn_like(y)
    y.backward(g)
    xc, wc = x.detach().cpu().requires_grad_(), w.detach().cpu().requires_grad_()
    yc = fp8.fp8_linear(xc, wc, recipe="mx")
    yc.backward(g.cpu())
    assert _rel(y.cpu(), yc) < 2e-2
    assert _rel(x.grad.cpu(), xc.grad) < 2e-2
    assert _rel(w.grad.cpu(), wc.grad) < 2e-2
    xd, wd = x.detach().double().requires_grad_(), w.detach().double().requires_grad_()
    yd = xd @ wd.t()
    yd.backward(g.double())
    errs = (_rel(y, yd), _rel(x.grad, xd.grad), _rel(w.grad, wd.grad))
    print(f"mxfp8 linear: rel err y / dx / dW = {errs[0]:.2e} / {errs[1]:.2e} / {errs[2]:.2e}")
    assert max(errs) < 0.06
