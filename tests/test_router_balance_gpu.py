"""The fused router kernel's auxiliary-loss path (``STATS`` / ``BALANCE`` instantiations of ``ops/csrc/router.cu``)
against an fp64 reference.  The forward's per-sequence statistics: exact selection counts and fp32-sum bounds on the score
and lse^2 sums at every experts-per-lane bucket, for softmax and sigmoid scores, for the batch losses' single sequence
(``num_seqs = 1``: no tokens, one, a few, several grid passes of tokens per warp), one-token sequences, sequences that end
inside a block and many short ones; bitwise-reproducible statistics.  The backward within one bf16 rounding of fp64 for
each term alone and together, both score functions and every option; a zero gradient bitwise equal to the plain backward;
refused operands; no host synchronisation; and ``route_topk`` and ``MoELayer`` routers on CUDA against the PyTorch path."""

import pytest
import torch

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24
W_TOK = 1e-3
SCORES = ["softmax", "sigmoid"]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from d9d_b200.kernel._native import native_ops

    return native_ops()


def _warps(T):
    """Warps of the plain kernels' grid for T tokens (blocks of 8 warps, at most 8 blocks per SM)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, min((T + 7) // 8, sms * 8)) * 8


def _balance_scores(x, score_function):
    if score_function == "softmax":
        return torch.softmax(x, -1)
    sig = torch.sigmoid(x)
    return sig / sig.sum(-1, keepdim=True)


def _reference_stats(logits, idx, B, score_function):
    x = logits.double()
    T, E = x.shape
    S = T // B
    s = _balance_scores(x, score_function)
    sel = idx.reshape(B, -1).cpu()
    counts = torch.zeros(B, E, dtype=torch.int64).scatter_add_(1, sel, torch.ones_like(sel))
    lse = torch.logsumexp(x, -1)
    return counts, s.reshape(B, S, E).sum(1), (lse * lse).reshape(B, S).sum(1), lse.reshape(B, S)


def _check_stats(ops, logits, k, B, score_function, bias=None, groups=(1, 1), renorm=True, scale=1.0):
    """Statistics of B sequences of T / B tokens (B = 1: the batch losses')."""
    T, E = logits.shape
    S = T // B
    idx, probs, counts, ssum, lse2 = ops.router_topk_fwd(logits, bias, k, renorm, score_function, *groups, scale, B)
    idx0, probs0, *none = ops.router_topk_fwd(logits, bias, k, renorm, score_function, *groups, scale, 0)
    assert torch.equal(idx, idx0) and torch.equal(probs, probs0)  # routing is untouched
    assert none == [None, None, None]  # no statistics without a sequence count
    rc, rs, rl, lse = _reference_stats(logits, idx, B, score_function)
    assert counts.dtype == torch.int32 and counts.shape == (B, E)
    assert torch.equal(counts.cpu().long(), rc)
    assert torch.equal(counts.sum(1).cpu(), torch.full((B,), S * k))
    per_warp = -(-T // _warps(T))  # tokens per warp in a block's range
    parts = -(-S // (8 * per_warp)) if T else 0
    terms = per_warp + 8 + parts  # per-warp, in-block and across-block fp32 additions
    score_err = 4e-6 if score_function == "softmax" else 1e-5  # approximate exp; sigmoid adds the normalising sum
    bound_s = (terms * EPS32 + score_err) * rs + 1e-30
    assert ((ssum.double() - rs).abs() <= bound_s).all(), (ssum.double() - rs).abs().max()
    if score_function == "softmax":
        bound_l = (terms * EPS32 + 4e-6) * rl + 2 * 4e-6 * lse.abs().sum(1) + 1e-30
        assert ((lse2.double() - rl).abs() <= bound_l).all(), (lse2.double() - rl).abs().max()
    else:
        assert not lse2.any()
    return idx, counts, ssum


# ---- forward statistics: the batch losses' single sequence ----

@pytest.mark.parametrize("E", [32, 64, 128, 256, 512, 1024, 200])
@pytest.mark.parametrize("k", [1, 2, 8])
def test_batch_statistics_at_every_bucket(ops, E, k):
    torch.manual_seed(E * 31 + k)
    for T in (0, 1, 7, 1000):
        logits = (torch.randn(T, E, device="cuda") * 2).bfloat16()
        _check_stats(ops, logits, k, 1, "softmax")


def test_batch_statistics_over_several_grid_passes(ops):
    T = 3 * _warps(1 << 30) + 37  # every warp of the capped grid makes four passes, the last one ragged
    torch.manual_seed(0)
    for E, k in ((128, 8), (1024, 32)):
        _check_stats(ops, (torch.randn(T, E, device="cuda") * 3).bfloat16(), k, 1, "softmax")


def test_batch_statistics_with_bias_and_groups(ops):
    torch.manual_seed(1)
    E = 256
    bias = torch.randn(E, device="cuda") * 0.01
    logits = torch.randn(3000, E, device="cuda").bfloat16()
    _check_stats(ops, logits, 8, 1, "softmax", bias=bias, groups=(8, 4), scale=2.5)
    _check_stats(ops, logits, 6, 1, "softmax", bias=bias, groups=(8, 3), renorm=False)


def test_batch_statistics_are_bitwise_reproducible(ops):
    T = 3 * _warps(1 << 30) + 37
    logits = torch.randn(T, 128, device="cuda").bfloat16()
    a = ops.router_topk_fwd(logits, None, 8, True, "softmax", 1, 1, 1.0, 1)
    b = ops.router_topk_fwd(logits, None, 8, True, "softmax", 1, 1, 1.0, 1)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---- forward statistics: several sequences ----

@pytest.mark.parametrize("E", [8, 32, 64, 128, 256, 512, 1024, 200])
@pytest.mark.parametrize("score_function", SCORES)
def test_sequence_statistics_at_every_bucket(ops, E, score_function):
    torch.manual_seed(E)
    k = min(8, E)
    # one token; one-token sequences; sequences ending inside a block (37 tokens); 200-token sequences; many short ones
    for T, S in ((1, 1), (96, 1), (37 * 5, 37), (1000, 200), (4096, 2)):
        logits = (torch.randn(T, E, device="cuda") * 2).bfloat16()
        _check_stats(ops, logits, k, T // S, score_function)


@pytest.mark.parametrize("score_function", SCORES)
def test_sequence_statistics_with_several_tokens_per_warp(ops, score_function):
    torch.manual_seed(0)
    S = _warps(1 << 30) + 37  # three sequences: every warp of the capped grid walks 4 tokens of its block's range
    for E, k in ((256, 8), (1024, 32)):
        _check_stats(ops, (torch.randn(3 * S, E, device="cuda") * 3).bfloat16(), k, 3, score_function)
    _check_stats(ops, (torch.randn(3 * S, 64, device="cuda") * 3).bfloat16(), 4, 1, score_function)


@pytest.mark.parametrize("score_function", SCORES)
def test_sequence_statistics_with_bias_groups_and_scaling(ops, score_function):
    torch.manual_seed(1)
    E = 256
    bias = torch.randn(E, device="cuda") * 0.01
    logits = torch.randn(4096, E, device="cuda").bfloat16()
    _check_stats(ops, logits, 8, 4, score_function, bias=bias, groups=(8, 4), scale=2.5)
    _check_stats(ops, logits, 6, 8, score_function, bias=bias, groups=(8, 3), renorm=False)


def test_no_tokens(ops):
    logits = torch.empty(0, 64, device="cuda").bfloat16()
    idx, probs, *none = ops.router_topk_fwd(logits, None, 4, True, "sigmoid", 1, 1, 1.0, 0)
    assert idx.shape == (0, 4) and probs.shape == (0, 4) and none == [None, None, None]
    _, _, counts, ssum, lse2 = ops.router_topk_fwd(logits, None, 4, True, "sigmoid", 1, 1, 1.0, 3)
    assert counts.shape == (3, 64) and not counts.any() and not ssum.any() and not lse2.any()
    dprobs = torch.empty(0, 4, device="cuda")
    for g in (torch.zeros(1, 64, device="cuda"), torch.zeros(3, 64, device="cuda")):
        assert ops.router_topk_bwd(logits, idx, dprobs, True, "sigmoid", 1.0, g, 0.0).shape == (0, 64)


@pytest.mark.parametrize("score_function", SCORES)
def test_sequence_statistics_are_bitwise_reproducible(ops, score_function):
    S = _warps(1 << 30) + 37
    logits = torch.randn(3 * S, 256, device="cuda").bfloat16()
    bias = torch.randn(256, device="cuda") * 0.01
    a = ops.router_topk_fwd(logits, bias, 8, True, score_function, 8, 4, 2.5, 3)
    b = ops.router_topk_fwd(logits, bias, 8, True, score_function, 8, 4, 2.5, 3)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---- backward ----

def _reference_dlogits(logits, idx, dprobs, renorm, scale, score_function, g, zc):
    """fp64 selection gradient and balance + z-loss gradient for g [B, E] (row t // (T / B) for token t)."""
    x = logits.double().requires_grad_()
    scores = torch.softmax(x, -1) if score_function == "softmax" else torch.sigmoid(x)
    sel = scores.gather(-1, idx)
    r = sel / (sel.sum(-1, keepdim=True) + 1e-20) if renorm else sel
    (r * scale * dprobs.double()).sum().backward()
    xd = x.detach()
    s = _balance_scores(xd, score_function)
    if score_function == "softmax":
        d = s
    else:
        sig = torch.sigmoid(xd)
        d = sig * (1 - sig) / sig.sum(-1, keepdim=True)
    gt = g.double().repeat_interleave(x.shape[0] // g.shape[0], 0)
    lse = torch.logsumexp(xd, -1)
    aux = d * (gt - (s * gt).sum(-1, keepdim=True)) + zc * lse[:, None] * s
    return x.grad, aux, d, lse


@pytest.mark.parametrize("E,k", [(32, 4), (128, 8), (200, 6), (1024, 32)])
@pytest.mark.parametrize("terms", ["lb", "z", "both"])
@pytest.mark.parametrize("renorm,scale", [(True, 1.0), (False, 2.5)])
def test_batch_backward_against_fp64(ops, E, k, terms, renorm, scale):
    torch.manual_seed(E + k)
    T = 777
    logits = (torch.randn(T, E, device="cuda") * 2).bfloat16()
    idx, _, counts, _, _ = ops.router_topk_fwd(logits, None, k, renorm, "softmax", 1, 1, scale, 1)
    dprobs = torch.randn(T, k, device="cuda")
    lb = 0.0 if terms == "z" else 0.05
    z = 0.0 if terms == "lb" else 1e-3
    w = 1.0  # a per-token weight that makes the auxiliary terms comparable with the selection gradient
    g = counts.float() * (w * lb * E / (k * T))
    zc = 2 * w * z
    got = ops.router_topk_bwd(logits, idx, dprobs, renorm, "softmax", scale, g, zc).double()
    main, aux, _, _ = _reference_dlogits(logits, idx, dprobs, renorm, scale, "softmax", g, zc)
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


@pytest.mark.parametrize("E,k", [(32, 4), (128, 8), (256, 8), (200, 6), (1024, 32)])
@pytest.mark.parametrize("score_function", SCORES)
@pytest.mark.parametrize("renorm,scale,with_batch", [(True, 1.0, False), (False, 2.5, False), (True, 2.5, True)])
def test_sequence_backward_against_fp64(ops, E, k, score_function, renorm, scale, with_batch):
    torch.manual_seed(E + k)
    S, B = 111, 7
    T = S * B
    logits = (torch.randn(T, E, device="cuda") * 2).bfloat16()
    idx, _, counts, _, _ = ops.router_topk_fwd(logits, None, k, renorm, score_function, 1, 1, scale, B)
    dprobs = torch.randn(T, k, device="cuda")
    w, coef = 1.0, 0.05  # a per-token weight that makes the balance term comparable with the selection gradient
    g = counts.float() * (w * coef * E / (k * S))
    zc = 0.0
    if with_batch and score_function == "softmax":  # + the batch load-balancing row and the z-loss
        g = g + counts.sum(0).float() * (w * 0.05 * E / (k * T))
        zc = 2 * w * 1e-3
    got = ops.router_topk_bwd(logits, idx, dprobs, renorm, score_function, scale, g, zc).double()
    main, aux, d, lse = _reference_dlogits(logits, idx, dprobs, renorm, scale, score_function, g, zc)
    ref = main + aux
    # bf16 output rounding + fp32 arithmetic (approximate exp / log / division: a few 1e-6 relative) on the terms that
    # the score derivative multiplies before they cancel: the selection gradient, g and s.g (over sum sigma for
    # sigmoid), and 2 w coef_z lse
    scores = torch.softmax(logits.double(), -1) if score_function == "softmax" else torch.sigmoid(logits.double())
    Ssel = scores.gather(-1, idx).sum(-1) if renorm else torch.ones(T, device="cuda", dtype=torch.float64)
    dsel = scores if score_function == "softmax" else scores * (1 - scores)
    gmax = g.abs().amax(1).double().repeat_interleave(S, 0)
    bal = 2 * gmax if score_function == "softmax" else 2 * gmax / torch.sigmoid(logits.double()).sum(-1)
    bound = (2.0 ** -8 * ref.abs() + 2e-5 * dsel * (2 * scale * dprobs.double().abs().sum(-1) / Ssel)[:, None]
             + 2e-5 * (dsel * bal[:, None] if score_function == "softmax" else d * 2 * gmax[:, None])
             + 2e-5 * zc * scores * lse.abs()[:, None] + 1e-12)
    assert ((got - ref).abs() <= bound).all(), ((got - ref).abs() - bound).max()
    assert aux.abs().max() > 2.0 ** -8 * ref.abs().max() * 1e-2  # the balance term is visible at this size


def test_zero_auxiliary_terms_reproduce_the_plain_backward(ops):
    torch.manual_seed(3)
    for E, k, renorm, scale in ((128, 8, True, 1.0), (64, 4, False, 2.5), (1024, 16, True, 1.0)):
        logits = torch.randn(500, E, device="cuda").bfloat16()
        idx, *_ = ops.router_topk_fwd(logits, None, k, renorm, "softmax", 1, 1, scale, 0)
        dprobs = torch.randn(500, k, device="cuda")
        plain = ops.router_topk_bwd(logits, idx, dprobs, renorm, "softmax", scale, None, 0.0)
        aux = ops.router_topk_bwd(logits, idx, dprobs, renorm, "softmax", scale, torch.zeros(1, E, device="cuda"), 0.0)
        assert torch.equal(plain, aux)


@pytest.mark.parametrize("score_function", SCORES)
def test_zero_balance_gradient_reproduces_the_plain_backward(ops, score_function):
    torch.manual_seed(3)
    for E, k, renorm, scale in ((128, 8, True, 1.0), (64, 4, False, 2.5), (1024, 16, True, 1.0)):
        logits = torch.randn(500, E, device="cuda").bfloat16()
        idx, *_ = ops.router_topk_fwd(logits, None, k, renorm, score_function, 1, 1, scale, 0)
        dprobs = torch.randn(500, k, device="cuda")
        plain = ops.router_topk_bwd(logits, idx, dprobs, renorm, score_function, scale, None, 0.0)
        seq = ops.router_topk_bwd(logits, idx, dprobs, renorm, score_function, scale, torch.zeros(5, E, device="cuda"), 0.0)
        assert torch.equal(plain, seq)


# ---- refusals ----

def test_bad_batch_operands_are_refused(ops):
    logits = torch.randn(16, 64, device="cuda").bfloat16()
    idx, *_ = ops.router_topk_fwd(logits, None, 4, True, "softmax", 1, 1, 1.0, 0)
    dprobs = torch.randn(16, 4, device="cuda")
    with pytest.raises(RuntimeError):
        ops.router_topk_bwd(logits, idx, dprobs, True, "softmax", 1.0, torch.zeros(1, 63, device="cuda"), 0.0)
    with pytest.raises(RuntimeError):
        ops.router_topk_bwd(logits, idx, dprobs, True, "softmax", 1.0,
                            torch.zeros(1, 64, device="cuda", dtype=torch.float64), 0.0)
    with pytest.raises(RuntimeError):
        ops.router_topk_bwd(logits, idx, dprobs[:, :3].contiguous(), True, "softmax", 1.0,
                            torch.zeros(1, 64, device="cuda"), 0.0)


def test_bad_sequence_operands_are_refused(ops):
    logits = torch.randn(16, 64, device="cuda").bfloat16()
    with pytest.raises(RuntimeError, match="divisor"):
        ops.router_topk_fwd(logits, None, 4, True, "sigmoid", 1, 1, 1.0, 5)
    with pytest.raises(RuntimeError, match="divisor"):
        ops.router_topk_fwd(logits, None, 4, True, "sigmoid", 1, 1, 1.0, -1)
    idx, *_ = ops.router_topk_fwd(logits, None, 4, True, "sigmoid", 1, 1, 1.0, 0)
    dprobs = torch.randn(16, 4, device="cuda")
    with pytest.raises(RuntimeError, match="divisor"):
        ops.router_topk_bwd(logits, idx, dprobs, True, "sigmoid", 1.0, torch.zeros(3, 64, device="cuda"), 0.0)
    with pytest.raises(RuntimeError):
        ops.router_topk_bwd(logits, idx, dprobs, True, "sigmoid", 1.0, torch.zeros(4, 64, device="cuda"), 1e-3)


# ---- route_topk and MoELayer ----

def test_route_topk_makes_no_host_synchronisation():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from d9d_b200.kernel.router import route_topk

    x = torch.randn(4096, 256, device="cuda").bfloat16().requires_grad_()
    bias = torch.randn(256, device="cuda") * 0.01
    dprobs = torch.randn(4096, 8, device="cuda")
    seq_sums, aux_sums = torch.zeros(2, device="cuda"), torch.zeros(3, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for score_function, batch in (("sigmoid", {}), ("softmax", {"load_balancing_coef": 0.01, "z_loss_coef": 1e-3,
                                                                    "aux_loss_sums": aux_sums})):
            _, p = route_topk(x, 8, True, bias, score_function, 8, 4, 2.5, token_loss_weight=W_TOK,
                              sequence_balance_coef=1e-2, sequence_length=1024, sequence_balance_sums=seq_sums, **batch)
            p.backward(dprobs)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert seq_sums[1].item() == pytest.approx(2 * W_TOK * 4096) and aux_sums[2].item() > 0


def test_route_topk_batch_losses_on_cuda_match_the_pytorch_path():
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


@pytest.mark.parametrize("score_function", SCORES)
def test_route_topk_sequence_loss_on_cuda_matches_the_pytorch_path(score_function):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from d9d_b200.kernel.router import route_topk

    torch.manual_seed(4)
    T, E, k, S = 2048, 128, 8, 256
    # distinct logits per row (multiples of 1/32, exact in bf16): no ties, so both paths select in the same order
    logits = (torch.argsort(torch.rand(T, E), dim=-1).float() / 32 - 2).bfloat16()
    dprobs = torch.randn(T, k)
    batch = {"load_balancing_coef": 0.05, "z_loss_coef": 1e-3} if score_function == "softmax" else {}
    out = {}
    for dev in ("cpu", "cuda"):
        x = logits.to(dev).clone().requires_grad_()
        sums = torch.zeros(2, device=dev)
        idx, p = route_topk(x, k, True, score_function=score_function, scaling_factor=2.5, token_loss_weight=W_TOK,
                            sequence_balance_coef=0.05, sequence_length=S, sequence_balance_sums=sums, **batch)
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
    for dev in ("cpu", "cuda"):  # bf16 logits: the PyTorch path on the CPU, the fused kernels with one sequence on CUDA
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


def test_deepseek_v3_moe_layer_on_cuda_matches_the_pytorch_path():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from d9d_b200.module.block.moe import MoELayer, RouterParameters

    torch.manual_seed(5)
    layer = MoELayer(hidden_dim=64, intermediate_dim_grouped=32, num_grouped_experts=16, top_k=4,
                     router_renormalize_probabilities=True,
                     router=RouterParameters(score_function="sigmoid", enable_expert_bias=True, num_expert_groups=4,
                                             topk_expert_groups=2, routed_scaling_factor=2.5))
    layer.reset_parameters()
    with torch.no_grad():
        layer.router.expert_bias.copy_(torch.randn(16) * 0.01)
    layer = layer.bfloat16()
    x = torch.randn(4, 128, 64).bfloat16()
    grads, sums = {}, {}
    for dev in ("cpu", "cuda"):  # bf16 logits: the PyTorch path on the CPU, the fused kernels per sequence on CUDA
        m = layer.to(dev)
        m.router.set_sequence_balance_loss(0.05, W_TOK)
        m.router.reset_aux_loss_sums()
        m.zero_grad()
        m(x.to(dev)).float().pow(2).mean().backward()
        grads[dev] = m.router.gate.weight.grad.float().cpu().clone()
        sums[dev] = m.router.sequence_balance_sums.cpu().clone()
    # bf16 gate GEMMs round differently on the two devices, so compare the gradient as a whole
    assert (grads["cuda"] - grads["cpu"]).norm() <= 0.05 * grads["cpu"].norm()
    torch.testing.assert_close(sums["cuda"], sums["cpu"], rtol=1e-2, atol=0)
