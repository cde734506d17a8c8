"""The fused router kernel's auxiliary-loss path (``AUX`` instantiations of ``ops/csrc/router.cu``) against an fp64
reference with per-element bounds: the forward statistics (exact counts, fp32-sum bounds for sum_t s and sum_t lse^2) at
every experts-per-lane bucket, several k and token counts up to several grid-stride passes per warp; the backward with
each term alone and both; bitwise determinism; and a router on CUDA against the PyTorch path."""

import pytest
import torch

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24
W_TOK = 1e-3


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from d9d_b200.kernel._native import native_ops

    return native_ops()


def _grid_tokens():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps = sms * 8 * 8  # capped grid: 8 blocks per SM, 8 warps per block
    return warps, 3 * warps + 37  # every warp makes three passes, plus a ragged tail


def _reference_stats(logits, idx, E):
    x = logits.double()
    s = torch.softmax(x, -1)
    lse = torch.logsumexp(x, -1)
    counts = torch.bincount(idx.reshape(-1).cpu(), minlength=E)
    return counts, s.sum(0), (lse * lse).sum(), s, lse


def _check_stats(ops, logits, k, bias=None, groups=(1, 1), renorm=True, scale=1.0):
    T, E = logits.shape
    idx, probs, counts, ssum, lse2 = ops.router_topk_aux_fwd(logits, bias, k, renorm, *groups, scale)
    idx0, probs0 = ops.router_topk_fwd(logits, bias, k, renorm, "softmax", *groups, scale)
    assert torch.equal(idx, idx0) and torch.equal(probs, probs0)  # routing is untouched
    rc, rs, rl, _, lse = _reference_stats(logits, idx, E)
    assert counts.dtype == torch.int32 and torch.equal(counts.cpu().long(), rc)
    warps, _ = _grid_tokens()
    parts = max(1, min((T + 7) // 8, warps // 8))
    terms = -(-T // warps) + 8 + parts  # per-warp, in-block and across-block fp32 additions
    bound_s = (terms * EPS32 + 4e-6) * rs + 1e-30
    assert ((ssum.double() - rs).abs() <= bound_s).all(), (ssum.double() - rs).abs().max()
    bound_l = (terms * EPS32 + 4e-6) * rl + 2 * 4e-6 * lse.abs().sum() + 1e-30
    assert abs(lse2.double().item() - rl.item()) <= bound_l, (lse2.item(), rl.item())
    return idx, counts, ssum, lse2


@pytest.mark.parametrize("E", [32, 64, 128, 256, 512, 1024, 200])
@pytest.mark.parametrize("k", [1, 2, 8])
def test_forward_statistics_at_every_bucket(ops, E, k):
    torch.manual_seed(E * 31 + k)
    for T in (0, 1, 7, 1000):
        logits = (torch.randn(T, E, device="cuda") * 2).bfloat16()
        _check_stats(ops, logits, k)


def test_forward_statistics_over_several_grid_passes(ops):
    _, T = _grid_tokens()
    torch.manual_seed(0)
    for E, k in ((128, 8), (1024, 32)):
        _check_stats(ops, (torch.randn(T, E, device="cuda") * 3).bfloat16(), k)


def test_forward_statistics_with_bias_and_groups(ops):
    torch.manual_seed(1)
    E = 256
    bias = torch.randn(E, device="cuda") * 0.01
    logits = torch.randn(3000, E, device="cuda").bfloat16()
    _check_stats(ops, logits, 8, bias=bias, groups=(8, 4), scale=2.5)
    _check_stats(ops, logits, 6, bias=bias, groups=(8, 3), renorm=False)


def test_forward_statistics_are_bitwise_reproducible(ops):
    _, T = _grid_tokens()
    logits = torch.randn(T, 128, device="cuda").bfloat16()
    a = ops.router_topk_aux_fwd(logits, None, 8, True, 1, 1, 1.0)
    b = ops.router_topk_aux_fwd(logits, None, 8, True, 1, 1, 1.0)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def _reference_dlogits(logits, idx, dprobs, renorm, scale, g, zc):
    x = logits.double().requires_grad_()
    s = torch.softmax(x, -1)
    sel = s.gather(-1, idx)
    r = sel / (sel.sum(-1, keepdim=True) + 1e-20) if renorm else sel
    (r * scale * dprobs.double()).sum().backward()
    lse = torch.logsumexp(x.detach(), -1)
    sd = s.detach()
    aux = sd * (g.double() - (sd @ g.double())[:, None]) + zc * lse[:, None] * sd
    return x.grad, aux


@pytest.mark.parametrize("E,k", [(32, 4), (128, 8), (200, 6), (1024, 32)])
@pytest.mark.parametrize("terms", ["lb", "z", "both"])
@pytest.mark.parametrize("renorm,scale", [(True, 1.0), (False, 2.5)])
def test_backward_against_fp64(ops, E, k, terms, renorm, scale):
    torch.manual_seed(E + k)
    T = 777
    logits = (torch.randn(T, E, device="cuda") * 2).bfloat16()
    idx, _, counts, _, _ = ops.router_topk_aux_fwd(logits, None, k, renorm, 1, 1, scale)
    dprobs = torch.randn(T, k, device="cuda")
    lb = 0.0 if terms == "z" else 0.05
    z = 0.0 if terms == "lb" else 1e-3
    w = 1.0  # a per-token weight that makes the auxiliary terms comparable with the selection gradient
    g = counts.float() * (w * lb * E / (k * T))
    zc = 2 * w * z
    got = ops.router_topk_aux_bwd(logits, idx, dprobs, renorm, scale, g, zc).double()
    main, aux = _reference_dlogits(logits, idx, dprobs, renorm, scale, g, zc)
    ref = main + aux
    # bf16 output rounding + fp32 arithmetic on the terms that s_e multiplies before they cancel: the selection
    # gradient (|ds| <= 2 scale sum|dr| / S, S the renormalising sum), g and s.g, and 2 w coef_z lse (approximate exp /
    # log: a few 1e-6 relative)
    s = torch.softmax(logits.double(), -1)
    S = s.gather(-1, idx).sum(-1) if renorm else torch.ones(T, device="cuda", dtype=torch.float64)
    lse = torch.logsumexp(logits.double(), -1)
    terms_t = 2 * scale * dprobs.double().abs().sum(-1) / S + 2 * g.abs().max().double() + zc * lse.abs()
    bound = 2.0 ** -8 * ref.abs() + 2e-5 * s * terms_t[:, None] + 1e-12
    assert ((got - ref).abs() <= bound).all(), ((got - ref).abs() - bound).max()
    assert aux.abs().max() > 2.0 ** -8 * ref.abs().max() * 1e-2  # the auxiliary term is visible at this size


def test_zero_auxiliary_terms_reproduce_the_plain_backward(ops):
    torch.manual_seed(3)
    for E, k, renorm, scale in ((128, 8, True, 1.0), (64, 4, False, 2.5), (1024, 16, True, 1.0)):
        logits = torch.randn(500, E, device="cuda").bfloat16()
        idx, _ = ops.router_topk_fwd(logits, None, k, renorm, "softmax", 1, 1, scale)
        dprobs = torch.randn(500, k, device="cuda")
        plain = ops.router_topk_bwd(logits, idx, dprobs, renorm, "softmax", scale)
        aux = ops.router_topk_aux_bwd(logits, idx, dprobs, renorm, scale, torch.zeros(E, device="cuda"), 0.0)
        assert torch.equal(plain, aux)


def test_bad_operands_are_refused(ops):
    logits = torch.randn(16, 64, device="cuda").bfloat16()
    idx, _ = ops.router_topk_fwd(logits, None, 4, True, "softmax", 1, 1, 1.0)
    dprobs = torch.randn(16, 4, device="cuda")
    with pytest.raises(RuntimeError):
        ops.router_topk_aux_bwd(logits, idx, dprobs, True, 1.0, torch.zeros(63, device="cuda"), 0.0)
    with pytest.raises(RuntimeError):
        ops.router_topk_aux_bwd(logits, idx, dprobs, True, 1.0, torch.zeros(64, device="cuda", dtype=torch.float64), 0.0)
    with pytest.raises(RuntimeError):
        ops.router_topk_aux_bwd(logits, idx, dprobs[:, :3].contiguous(), True, 1.0, torch.zeros(64, device="cuda"), 0.0)


def test_route_topk_on_cuda_matches_the_pytorch_path():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from d9d_b200.kernel.router import route_topk

    torch.manual_seed(4)
    T, E, k = 2048, 128, 8
    # distinct logits per row (multiples of 1/32, exact in bf16): no ties, so both paths select in the same order
    logits = (torch.argsort(torch.rand(T, E), dim=-1).float() / 32 - 2).bfloat16()
    dprobs = torch.randn(T, k)
    out = {}
    for dev in ("cpu", "cuda"):
        x = logits.to(dev).clone().requires_grad_()
        sums = torch.zeros(3, device=dev)
        idx, p = route_topk(x, k, True, load_balancing_coef=0.05, z_loss_coef=1e-3, token_loss_weight=W_TOK, aux_loss_sums=sums)
        (p * dprobs.to(dev)).sum().backward()
        out[dev] = (idx.cpu(), x.grad.float().cpu(), sums.cpu())
    assert torch.equal(out["cpu"][0], out["cuda"][0])
    torch.testing.assert_close(out["cuda"][1], out["cpu"][1], rtol=2 ** -7, atol=1e-6)
    torch.testing.assert_close(out["cuda"][2], out["cpu"][2], rtol=1e-5, atol=0)


def test_moe_layer_router_on_cuda_matches_the_pytorch_path():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from d9d_b200.module.block.moe import MoELayer

    torch.manual_seed(5)
    layer = MoELayer(hidden_dim=64, intermediate_dim_grouped=32, num_grouped_experts=16, top_k=4,
                     router_renormalize_probabilities=True)
    layer.reset_parameters()
    layer = layer.bfloat16()
    x = torch.randn(2, 128, 64).bfloat16()
    grads, sums = {}, {}
    for dev in ("cpu", "cuda"):  # bf16 logits: the PyTorch path on the CPU, the fused AUX kernels on CUDA
        m = layer.to(dev)
        m.router.set_aux_loss(0.05, 1e-3, W_TOK)
        m.router.reset_aux_loss_sums()
        m.zero_grad()
        m(x.to(dev)).float().pow(2).mean().backward()
        grads[dev] = m.router.gate.weight.grad.float().cpu().clone()
        sums[dev] = m.router.aux_loss_sums.cpu().clone()
    # bf16 gate GEMMs round differently on the two devices, so compare the gradient as a whole
    assert (grads["cuda"] - grads["cpu"]).norm() <= 0.05 * grads["cpu"].norm()
    torch.testing.assert_close(sums["cuda"], sums["cpu"], rtol=1e-2, atol=0)
