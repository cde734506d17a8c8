"""The regularised fused linear cross-entropy on the GPU: label smoothing and the z-loss.

The kernel ops ``ce_forward_reg`` (nll, lse, target logit and the row's logit sum) and ``ce_dlogits_reg`` are checked per
element against an fp64 reference with error bounds in the style of ``test_gemm_variants_gpu._check_ce``, in both CTA
modes, through the TMA and the direct-store (canaried) epilogue, with bias, soft-cap and a column offset, and with every
row ignored.  The public function is checked against fp64 autograd of ``F.cross_entropy(..., label_smoothing) + zeta
lse^2`` on materialised logits.  Runs are bitwise reproducible, make no host synchronisation, and with both coefficients
0 launch only the plain CE kernels.
"""

import re

import pytest
import torch
import torch.nn.functional as F

from d9d_b200.kernel.cce import linear_cross_entropy
from tests.gemm_reference import U_BF16, Canaried, assert_within, ck

pytestmark = pytest.mark.gpu

DEV = "cuda"
REGS = [(0.1, 1e-4), (0.1, 0.1), (1.0, 1e-4), (1.0, 0.1)]  # (label_smoothing, z_loss_coef)


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _reference(h, w, tgt, bias, softcap, col_offset, ignore=-100):
    z = h.double() @ w.double().t()
    S = h.double().abs() @ w.double().abs().t()
    if bias is not None:
        z = z + bias.double()
    dz = torch.ones_like(z)
    if softcap > 0:
        th = torch.tanh(z / softcap)
        z, dz = softcap * th, 1 - th * th
    lse = torch.logsumexp(z, -1)
    rel = tgt - col_offset
    inside = (tgt != ignore) & (rel >= 0) & (rel < w.shape[0])
    tl = torch.where(inside, z.gather(1, rel.clamp(0, w.shape[0] - 1)[:, None])[:, 0], torch.zeros_like(lse))
    nll = torch.where(tgt == ignore, torch.zeros_like(lse), lse - tl)
    return z, dz, S, lse, tl, nll, inside


def _check_reg(ops, T, V, K, eps, zeta, *, pair_mode, tma, bias=False, softcap=0.0, col_offset=0, all_ignored=False):
    h = (torch.randn(T, K, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(V, K, device=DEV) * 0.1).bfloat16()
    b = torch.randn(V, device=DEV) * 0.5 if bias else None
    num_classes = V + col_offset + (40 if col_offset else 0)  # the slice is part of a larger classifier when offset
    tgt = torch.randint(0, num_classes, (T,), device=DEV)
    for i, c in enumerate([0, V - 1, (V - 1) // 256 * 256 + (V - 1) % 256 // 2]):  # first, last, inside the last tile
        if i < T:
            tgt[i] = c + col_offset
    tgt[4::7] = -100
    if all_ignored:
        tgt[:] = -100
    prev = ops.gemm_set_pair_mode(pair_mode)
    try:
        nll, lse, tl, zsum = ops.ce_forward_reg(h, w, tgt, -100, b, softcap, col_offset)
        z, dz, S, rlse, rtl, rnll, inside = _reference(h, w, tgt, b, softcap, col_offset)
        n_tiles = (V + 255) // 256
        e_z = ck(K) * S.max(-1).values + 2.0**-20 * (1 + z.abs().max(-1).values) + (softcap * 2.0**-18 if softcap else 0.0)
        e_lse = e_z + (64 + n_tiles) * 2.0**-23 + 2.0**-19 * (1 + rlse.abs())
        assert_within(lse, rlse, e_lse, "lse")
        assert_within(tl, rtl, torch.where(inside, e_z, 0.0), "target logit")
        assert_within(nll, rnll, torch.where(tgt == -100, 0.0, e_lse + e_z), "nll")
        # fp32 sum: 64 terms per thread, two quad shuffles, then the tiles in order
        e_sum = V * e_z + (66 + n_tiles) * 2.0**-23 * z.abs().sum(-1)
        assert_within(zsum, z.sum(-1), e_sum, "logit sum")

        g = torch.rand(T, device=DEV)
        out = Canaried(T, V, torch.bfloat16, tma=tma, device=DEV)
        ops.ce_dlogits_reg(h, w, tgt, rlse.float(), g, out.view, -100, zeta, eps, num_classes, b, softcap, col_offset)
        p = torch.exp(z - rlse.double()[:, None])
        scale = (1 + 2 * zeta * rlse)[:, None]
        gv = (g.double() * (tgt != -100))[:, None]
        onehot = torch.zeros_like(p)
        rows = inside.nonzero()[:, 0]
        onehot[rows, tgt[rows] - col_offset] = 1
        terms = scale.abs() * p + (1 - eps) * onehot + eps / num_classes
        ref = gv * (scale * p - (1 - eps) * onehot - eps / num_classes) * dz
        bound = (U_BF16 * ref.abs() + gv * dz * scale.abs() * p * (e_z[:, None] + 2.0**-19 * (1 + (z - rlse[:, None]).abs()))
                 + gv * dz * terms * 2.0**-21)
        if softcap:
            bound = bound + gv * terms * 2.0**-16
        assert_within(out.view, ref, bound, "dlogits")
        out.assert_untouched()
    finally:
        ops.gemm_set_pair_mode(prev)


@pytest.mark.parametrize("eps,zeta", REGS)
@pytest.mark.parametrize("pair_mode", [0, 1])
@pytest.mark.parametrize("V", [1, 255, 257, 50257])
@pytest.mark.parametrize("T", [1, 129, 1000])
@pytest.mark.parametrize("tma", [True, False])
def test_regularised_ce_ops(ops, eps, zeta, pair_mode, V, T, tma):
    _check_reg(ops, T, V, 136, eps, zeta, pair_mode=pair_mode, tma=tma)


@pytest.mark.parametrize("eps,zeta", REGS)
@pytest.mark.parametrize("pair_mode", [0, 1])
@pytest.mark.parametrize("V", [257, 1500])
def test_regularised_ce_ops_bias_softcap_slice(ops, eps, zeta, pair_mode, V):
    _check_reg(ops, 1000, V, 128, eps, zeta, pair_mode=pair_mode, tma=True, bias=True, softcap=8.0, col_offset=300)


@pytest.mark.parametrize("pair_mode", [0, 1])
def test_regularised_ce_ops_all_rows_ignored(ops, pair_mode):
    _check_reg(ops, 1000, 300, 128, 0.1, 0.1, pair_mode=pair_mode, tma=False, all_ignored=True)


def test_regularised_ce_ops_refuse_bad_operands(ops):
    T, V, K = 64, 300, 128
    h = torch.randn(T, K, device=DEV).bfloat16()
    w = torch.randn(V, K, device=DEV).bfloat16()
    tgt = torch.randint(0, V, (T,), device=DEV)
    lse, g = torch.zeros(T, device=DEV), torch.ones(T, device=DEV)
    out = torch.full((T, V), 3.0, device=DEV, dtype=torch.bfloat16)
    good = dict(z_loss_coef=1e-4, label_smoothing=0.1, num_classes=V)

    def bwd(**kw):
        a = dict(h=h, w=w, target=tgt, lse=lse, grad=g, out=out, ignore_index=-100) | good | kw
        ops.ce_dlogits_reg(a["h"], a["w"], a["target"], a["lse"], a["grad"], a["out"], a["ignore_index"], a["z_loss_coef"],
                           a["label_smoothing"], a["num_classes"], a.get("bias"), a.get("softcap", 0.0), a.get("col_offset", 0))

    for kw, match in [({"label_smoothing": -0.1}, "label_smoothing"), ({"label_smoothing": 1.5}, "label_smoothing"),
                      ({"label_smoothing": float("nan")}, "label_smoothing"), ({"z_loss_coef": -1.0}, "z_loss_coef"),
                      ({"z_loss_coef": float("inf")}, "z_loss_coef"), ({"num_classes": V - 1}, "num_classes"),
                      ({"col_offset": 5}, "num_classes"), ({"lse": torch.zeros(T + 1, device=DEV)}, "lse"),
                      ({"grad": g.double()}, "fp32"), ({"target": tgt.int()}, "int64"), ({"h": h.float()}, "bf16"),
                      ({"out": out[:, :-1]}, "out"), ({"bias": torch.zeros(V + 1, device=DEV)}, "bias"),
                      ({"softcap": float("nan")}, "softcap"), ({"w": w[:, :120].contiguous()}, "shape")]:
        with pytest.raises(RuntimeError, match=match):
            bwd(**kw)
    with pytest.raises(RuntimeError, match="int64"):
        ops.ce_forward_reg(h, w, tgt.int(), -100)
    with pytest.raises(RuntimeError, match="bias"):
        ops.ce_forward_reg(h, w, tgt, -100, torch.zeros(V, device=DEV, dtype=torch.bfloat16))
    assert (out == 3.0).all()


# ----------------------------------------------------------------------------- the public function
def _rel_err(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-12)).item()


@pytest.mark.parametrize("eps,zeta", [(0.1, 0.0), (0.0, 0.1), (0.1, 1e-4), (1.0, 0.1)])
@pytest.mark.parametrize("sizes,budget", [((4000,), 1 << 30), ((3000, 24), 1 << 30), ((1000, 520, 8), 512 * 1024 * 2)])
@pytest.mark.parametrize("fused_wgrad", [False, True])
@pytest.mark.parametrize("softcap,with_bias", [(None, False), (8.0, True)])
def test_public_function_against_fp64_autograd(monkeypatch, eps, zeta, sizes, budget, fused_wgrad, softcap, with_bias):
    from d9d_b200.kernel import _native
    from d9d_b200.kernel.cce import main as cce

    monkeypatch.setattr(cce, "_CHUNK_BYTES", budget)
    T, K = 640, 256
    e = (torch.randn(T, K, device=DEV) * 0.5).bfloat16().requires_grad_()
    ws = [(torch.randn(s, K, device=DEV) * 0.1).bfloat16().requires_grad_() for s in sizes]
    bias = (torch.randn(sum(sizes), device=DEV) * 0.3).requires_grad_() if with_bias else None
    tgt = torch.randint(0, sum(sizes), (T,), device=DEV)
    tgt[::9] = -100
    tgt[3] = sum(sizes) - 1
    if fused_wgrad:
        for w in ws:
            w.grad_dtype = torch.float32
            w.grad = torch.full(w.shape, 0.5, device=DEV, dtype=torch.float32)
            setattr(w, _native.FUSED_WGRAD_ATTR, True)
    e64 = e.detach().double().requires_grad_()
    w64 = [w.detach().double().requires_grad_() for w in ws]
    b64 = bias.detach().double().requires_grad_() if with_bias else None
    z = e64 @ torch.cat(w64).t()
    if with_bias:
        z = z + b64
    if softcap:
        z = softcap * torch.tanh(z / softcap)
    lse = torch.logsumexp(z, -1)
    ref_t = F.cross_entropy(z, tgt, reduction="none", label_smoothing=eps) + zeta * lse * lse * (tgt != -100)
    n = (tgt != -100).sum()
    with torch.no_grad():
        for reduction, ref in (("sum", ref_t.sum()), ("mean", ref_t.sum() / n)):
            loss = cce.linear_cross_entropy(e, ws, tgt, bias=bias, softcap=softcap, reduction=reduction,
                                            label_smoothing=eps, z_loss_coef=zeta)
            assert torch.allclose(loss.double(), ref, rtol=2e-3, atol=2e-3), reduction
    loss = cce.linear_cross_entropy(e, ws, tgt, bias=bias, softcap=softcap, reduction="none", label_smoothing=eps,
                                    z_loss_coef=zeta)
    assert torch.allclose(loss.double(), ref_t, rtol=2e-3, atol=2e-3)
    wgt = torch.rand(T, device=DEV, dtype=torch.float64)  # a non-uniform upstream gradient
    (loss.double() * wgt).sum().backward()
    (ref_t * wgt).sum().backward()
    assert _rel_err(e.grad, e64.grad) < 2e-2
    for w, r in zip(ws, w64):
        assert _rel_err(w.grad.float() - (0.5 if fused_wgrad else 0.0), r.grad) < 2e-2
    if with_bias:
        assert _rel_err(bias.grad, b64.grad) < 2e-2


def _problem(T=1000, K=256, sizes=(3000, 24)):
    g = torch.Generator(device=DEV).manual_seed(0)
    e = (torch.randn(T, K, device=DEV, generator=g) * 0.5).bfloat16().requires_grad_()
    ws = [(torch.randn(s, K, device=DEV, generator=g) * 0.1).bfloat16().requires_grad_() for s in sizes]
    tgt = torch.randint(0, sum(sizes), (T,), device=DEV, generator=g)
    tgt[::7] = -100
    return e, ws, tgt


def _run(e, ws, tgt, **kw):
    for t in (e, *ws):
        t.grad = None
    loss = linear_cross_entropy(e, ws, tgt, reduction="none", **kw)
    loss.sum().backward()
    return [loss.detach().clone(), e.grad.clone(), *[w.grad.clone() for w in ws]]


def test_two_runs_are_bitwise_equal():
    e, ws, tgt = _problem()
    sums = [torch.zeros(3, device=DEV) for _ in range(2)]
    a = _run(e, ws, tgt, label_smoothing=0.1, z_loss_coef=1e-4, loss_sums=sums[0])
    b = _run(e, ws, tgt, label_smoothing=0.1, z_loss_coef=1e-4, loss_sums=sums[1])
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert torch.equal(sums[0], sums[1]) and sums[0][2].item() == (tgt != -100).sum().item()


def test_no_host_synchronisation():
    e, ws, tgt = _problem()
    sums = torch.zeros(3, device=DEV)
    _run(e, ws, tgt, label_smoothing=0.1, z_loss_coef=1e-4, loss_sums=sums)  # warm up (first use loads the extension)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = linear_cross_entropy(e, ws, tgt, reduction="mean", label_smoothing=0.1, z_loss_coef=1e-4, loss_sums=sums)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def _ce_epilogues(prof):
    """Epilogue numbers of the CE GEMM instances the profile saw (names demangled or not)."""
    epis = set()
    for ev in prof.events():
        m = re.search(r"gemm_kernel<0, 256, false, false, (\d+), 0,", ev.name) or re.search(
            r"gemm_kernelILi0ELi256ELb0ELb0ELi(\d+)ELi0E", ev.name)
        if m:
            epis.add(int(m.group(1)))
        if "ce_finalize" in ev.name:
            epis.add("finalize_zsum" if "zsum" in ev.name else "finalize")
    return epis


def test_zero_coefficients_launch_only_the_plain_kernels_and_are_bitwise_the_plain_call():
    from torch.profiler import ProfilerActivity, profile

    e, ws, tgt = _problem()
    plain = _run(e, ws, tgt)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        zero = _run(e, ws, tgt, label_smoothing=0.0, z_loss_coef=0.0)
        torch.cuda.synchronize()
    for x, y in zip(plain, zero):
        assert torch.equal(x, y)
    assert _ce_epilogues(prof) == {4, 5, "finalize"}  # EPI_CE_LSE and EPI_CE_DLOGITS only
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run(e, ws, tgt, label_smoothing=0.1, z_loss_coef=1e-4)
        torch.cuda.synchronize()
    assert _ce_epilogues(prof) == {6, 7, "finalize_zsum"}  # EPI_CE_LSE_SUM and EPI_CE_DLOGITS_REG
